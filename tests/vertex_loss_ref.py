"""Float64 references, operand generators and exactness checks for the training step's vertex targets and vertex loss
(csrc/train_targets.cu): the 2-D centre targets (pixel_targets), the VERTEX_REG_3D targets (pixel_targets_3d), the
multi-instance targets (k_vertex_targets_instances), the fused loss of either mode (k_vertex_loss_fused) and the pose blob /
meta packing (k_pack_pose_meta).

Why the comparisons can be bit for bit:
- Vertex values.  The 1/8-resolution vertex channels lie on a dyadic grid `unit` and the biases on unit / 256, so every
  value of up8(lowres) + bias is a multiple of unit / 256; while the sum of the magnitudes of its terms stays below
  2^24 unit / 256 (the bit budget of tests/heads_ref.py) every fp32 operation of up8_value is exact, including its fmaf
  blends, and the kernel's value equals heads_ref's float64 one.
- 2-D direction channels: (float)(dx / (sqrt(dx^2 + dy^2) + 1e-10)) with dx, dy formed in double.  Double `/` and `sqrt`
  are correctly rounded on the device and in numpy, and nvcc contracts dx*dx + dy*dy into DMUL + DFMA.  Centres here are
  float32 multiples of 2^-12 within 2^11 of every pixel, so dx^2 and dx^2 + dy^2 are exact in double and the contraction
  cannot change the result (check_square_sums_exact asserts it on the generated centres).
- log z: the device's double `log` is within 1 ulp, not correctly rounded.  check_log_midpoints requires float64 log(z) of
  every distinct z to lie more than MIDPOINT_ULPS double ulps from an fp32 rounding midpoint, so that both the device's and
  numpy's value round to the same float32.  Generators draw z from LOGZ_TABLE, which passes.
- 3-D targets: coord_scale / coord_target (csrc/heads_common.cuh) restated op by op in float32 (heads_ref.coord_scale).
  The generated extents and object coordinates are not dyadic, so these operations round and a fused or reordered
  formula moves targets by an ulp (test_vertex_loss_exact_cpu.py shows it on the generated operands).
- The per-pixel smooth-L1 term (sl1_term) restated in numpy float32, one rounding per operation.

Contractions in the cross-compiled library (cuobjdump -sass of train_targets.o, sm_90a), and how the references handle them:
- dx*dx + dy*dy -> DMUL + DFMA in k_vertex_targets_sparse, k_vertex_targets_instances and k_vertex_loss_fused<false>:
  exact on the generated centres (above).
- span = vmax - vmin in coord_scale -> FMUL (vmin = e * -0.5) + FFMA(e, 0.5, -vmin): e * 0.5 is exact for normal e, so the
  fused result equals the rounded float32 subtraction of the reference.
- deconv_w's (float)x * 0.125f - 0.9375f -> FFMA: the product is exact, so the result is the same.
- sw += 3.0 * w_inside -> DFMA: 3 w is exact in double and so is every partial sum of the weights.
- up8_vblend / up8_hblend are fmaf by source: exact on the dyadic grid (above).
- sl1_term and coord_target compile to FADD / FMUL / FSETP only: no FFMA, so the numpy float32 restatements hold as written.
The division and square-root subroutines contain FFMA / DFMA by construction; they are correctly rounded.

The loss: out[0] = (float)(sum_terms / (sum_w + 1e-10)) with the terms accumulated in double in an order this module does
not assume.  loss_vertex forms the exact sum S of the float32 terms (exact_sum), bounds any double-accumulation order by
|error| <= N 2^-53 sum |term| (N: terms plus the kernel's grid of partial sums), adds the quotient's rounding, and raises
Straddle unless the whole interval rounds to one float32.  The weight sum 3 w_inside count is exact.
"""
import math
from fractions import Fraction

import numpy as np
import torch

from tests import heads_ref as R
from tests.heads_ref import BudgetExceeded, check_budget, check_grid  # noqa: F401

f32 = np.float32
LOSS_BLOCKS, LOSS_THREADS = R.NUM_SMS * 4, 256           # kLossBlocks x kLossThreads of the fused losses
MIDPOINT_ULPS = 4
LOGZ_TABLE = np.array([0.5, 0.75, 0.9, 1.0, 1.25, 1.5, 2.0], np.float32)   # log(z) far from fp32 midpoints (checked)


class MidpointTooClose(AssertionError):
    """float64 log(z) is too close to an fp32 rounding midpoint: a 1-ulp error of the device log could round differently."""


class Straddle(AssertionError):
    """The loss's error interval contains an fp32 rounding boundary: the kernel's value is not determined."""


# ---------------------------------------------------------------------------------------------------------------------
# exactness preconditions
# ---------------------------------------------------------------------------------------------------------------------
def near_f32_midpoint(L, ulps=MIDPOINT_ULPS):
    """True where float64 values L lie within `ulps` double ulps of a midpoint between two adjacent float32 values."""
    L = np.asarray(L, np.float64)
    r = L.astype(np.float32)
    r64 = r.astype(np.float64)
    toward = np.where(L > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
    nb = np.nextafter(r, toward).astype(np.float64)
    mid = (r64 + nb) / 2                                   # exact in double
    return np.abs(L - mid) <= ulps * np.spacing(np.abs(L))


def check_log_midpoints(z, ulps=MIDPOINT_ULPS):
    """float32 log targets of the positive float32 values z (any shape); raises MidpointTooClose if float64 log of a
    distinct z lies within `ulps` double ulps of an fp32 midpoint."""
    z = np.asarray(z, np.float32)
    u = np.unique(z)
    bad = u[near_f32_midpoint(np.log(u.astype(np.float64)), ulps)]
    if bad.size:
        raise MidpointTooClose(f"log z of {bad[:5].tolist()} within {ulps} double ulps of an fp32 midpoint")
    return np.log(z.astype(np.float64)).astype(np.float32)


def check_square_sums_exact(cx, cy, H, W):
    """Centre coordinates (float32) are multiples of 2^-12 and within 2^11 of every pixel of an H x W image: then dx, dy
    have at most 23 significant bits, dx^2 + dy^2 < 2^23 is a multiple of 2^-24, and it is exact in double with or without
    a fused multiply-add."""
    for name, c, n in (("cx", cx, W), ("cy", cy, H)):
        c = np.asarray(c, np.float32).astype(np.float64)
        assert np.all(c * 4096 == np.round(c * 4096)), f"{name}: not a multiple of 2^-12"
        assert np.all((c > -2048 + n) & (c < 2048)), f"{name}: farther than 2^11 from a pixel of a {H}x{W} image"


def exact_sum(x):
    """Exact sum of float32 values as a Fraction: each value is M 2^(e-24) with an integer M below 2^24, the M of one
    exponent are summed in int64 (exact below 2^39 values), and the per-exponent sums are combined exactly."""
    x = np.asarray(x, np.float32).ravel().astype(np.float64)
    m, e = np.frexp(x)
    M = (m * (1 << 24)).astype(np.int64)
    assert np.all(M.astype(np.float64) == m * (1 << 24)) and x.size < (1 << 39)
    order = np.argsort(e, kind="stable")
    e, M = e[order], M[order]
    if x.size == 0:
        return Fraction(0)
    starts = np.flatnonzero(np.r_[True, e[1:] != e[:-1]])
    sums = np.add.reduceat(M, starts)
    total = Fraction(0)
    for ex, s in zip(e[starts].tolist(), sums.tolist()):
        total += Fraction(int(s)) * (Fraction(2) ** (int(ex) - 24))
    return total


def _f32_of(q):
    """fp32 round-to-nearest of a double q."""
    return np.float32(np.float64(q))


# ---------------------------------------------------------------------------------------------------------------------
# targets: per-pixel form (listed [B,H,W] bool, cls [B,H,W] int64, t [B,H,W,3] float32) and the dense blobs
# ---------------------------------------------------------------------------------------------------------------------
def _listed(label, z_of_class, C):
    """label l in 1..C-1 whose class z (float32, [B,C]) is > 0 (NaN is not)."""
    label = np.asarray(label).astype(np.int64)
    inr = (label > 0) & (label < C)
    cls = np.where(inr, label, 0)
    z = np.take_along_axis(np.asarray(z_of_class, np.float32), cls.reshape(cls.shape[0], -1), 1).reshape(cls.shape)
    listed = inr & (z > 0)
    return listed, np.where(listed, cls, 0), z


def directions(cx, cy, H, W):
    """(float)(dx / (sqrt(dx^2 + dy^2) + 1e-10)), the same for dy, toward float32 centres cx, cy [B,H,W] from the pixel
    grid, in float64 with one float32 rounding (pixel_targets)."""
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    dx = np.asarray(cx, np.float32).astype(np.float64) - xs
    dy = np.asarray(cy, np.float32).astype(np.float64) - ys
    nrm = np.sqrt(dx * dx + dy * dy) + 1e-10
    return (dx / nrm).astype(np.float32), (dy / nrm).astype(np.float32)


def targets_2d(label, centers):
    """pixel_targets for every pixel: label [B,H,W], centers [B,C,3] float32."""
    centers = np.asarray(centers, np.float32)
    B, H, W = np.asarray(label).shape
    C = centers.shape[1]
    listed, cls, z = _listed(label, centers[..., 2], C)
    cen = np.take_along_axis(centers, cls.reshape(B, -1, 1), 1).reshape(B, H, W, 3)
    cx, cy = np.where(listed, cen[..., 0], 0), np.where(listed, cen[..., 1], 0)
    check_square_sums_exact(cx[listed], cy[listed], H, W)
    t = np.zeros((B, H, W, 3), np.float32)
    t[..., 0], t[..., 1] = directions(cx, cy, H, W)
    t[listed, 2] = check_log_midpoints(z[listed])
    t[~listed] = 0
    return listed, cls, t


def targets_3d(label, vertmap, centers, extents):
    """pixel_targets_3d for every pixel: t = (a v rounded) + b rounded per axis, (a, b) = coord_scale(extents[cls])."""
    centers = np.asarray(centers, np.float32)
    C = centers.shape[1]
    listed, cls, _ = _listed(label, centers[..., 2], C)
    ab = R.coord_scale(torch.as_tensor(np.asarray(extents, np.float32))).numpy()     # [C,3,2] float32
    a, b = ab[cls, :, 0], ab[cls, :, 1]
    t = ((a * np.asarray(vertmap, np.float32)).astype(np.float32) + b).astype(np.float32)
    t[~listed] = 0
    return listed, cls, t


def targets_instances(label, mask, instances, C):
    """k_vertex_targets_instances: pixel (label l in 1..C-1, mask m) belongs to the LAST instance row i of its image with
    z > 0, (int)cls == l and (int)mask_id == m; z <= 0 (or NaN) marks an unused slot."""
    label, mask = np.asarray(label).astype(np.int64), np.asarray(mask).astype(np.int64)
    inst = np.asarray(instances, np.float32)
    B, H, W = label.shape
    inr = (label > 0) & (label < C)
    hit = np.full((B, H, W), -1, np.int64)
    for i in range(inst.shape[1]):
        r = inst[:, i]
        use = (r[:, 4] > 0)[:, None, None] & (label == r[:, 0].astype(np.int64)[:, None, None]) \
            & (mask == r[:, 1].astype(np.int64)[:, None, None])
        hit = np.where(inr & use, i, hit)
    listed = hit >= 0
    row = np.take_along_axis(inst, np.maximum(hit, 0).reshape(B, -1, 1), 1).reshape(B, H, W, 5)
    cx, cy = np.where(listed, row[..., 2], 0), np.where(listed, row[..., 3], 0)
    check_square_sums_exact(cx[listed], cy[listed], H, W)
    t = np.zeros((B, H, W, 3), np.float32)
    t[..., 0], t[..., 1] = directions(cx, cy, H, W)
    t[listed, 2] = check_log_midpoints(row[listed, 4])
    t[~listed] = 0
    return listed, np.where(listed, label, 0), t


def dense(listed, cls, t, C, w_inside):
    """The materialised (vertex_targets, vertex_weights) [B,H,W,3C] float32 of per-pixel targets."""
    B, H, W = listed.shape
    tg = np.zeros((B, H, W, C, 3), np.float32)
    wt = np.zeros((B, H, W, C, 3), np.float32)
    b, y, x = np.nonzero(listed)
    tg[b, y, x, cls[b, y, x]] = t[b, y, x]
    wt[b, y, x, cls[b, y, x]] = np.float32(w_inside)
    return tg.reshape(B, H, W, 3 * C), wt.reshape(B, H, W, 3 * C)


# ---------------------------------------------------------------------------------------------------------------------
# vertex values and the loss
# ---------------------------------------------------------------------------------------------------------------------
def own_vertex_values(lowres, bias_v, cls, C, unit, chunk=4):
    """The three vertex values of each pixel's class, up8(lowres[..., C:]) + bias_v, in float64 on lowres' device, images in
    chunks.  lowres's vertex channels on the grid `unit`, bias_v on unit / 256.  Returns (float32 numpy [B,H,W,3],
    budget); the budget is the largest sum of |terms| in units of unit / 256 (BudgetExceeded at 2^24)."""
    lv = lowres[..., C:]
    check_grid("lowres (vertex)", lv, unit)
    check_grid("bias_vertex", bias_v, unit / 256)
    bias = bias_v.double().to(lowres.device)
    cls_t = torch.as_tensor(cls).to(lowres.device)
    out, budget = [], 0.0
    for i in range(0, lv.shape[0], chunk):
        part = lv[i:i + chunk]
        budget = max(budget, check_budget("up8 vertex", (R.up(part.abs(), 8) + bias.abs()).amax() / (unit / 256)))
        v = (R.up(part, 8) + bias).view(*part.shape[:1], 8 * part.shape[1], 8 * part.shape[2], C, 3)
        idx = cls_t[i:i + chunk].long()[..., None, None].expand(*v.shape[:3], 1, 3)
        own = v.gather(3, idx)[..., 0, :]
        assert bool((own.float().double() == own).all())
        out.append(own.float().cpu().numpy())
    return np.concatenate(out), budget


def sl1_terms(pred, targ, w_inside, sigma):
    """sl1_term in float32, one rounding per operation: diff = w (pred - targ); |diff| < 1 / sigma^2 ? diff^2 (sigma^2 / 2)
    : |diff| - 0.5 / sigma^2, with sigma^2 = sigma * sigma rounded (the entry point's sigma * sigma)."""
    s2 = f32(sigma) * f32(sigma)
    diff = f32(w_inside) * (np.asarray(pred, np.float32) - np.asarray(targ, np.float32))
    ad = np.abs(diff)
    return np.where(ad < f32(1) / s2, (diff * diff) * (s2 * f32(0.5)), ad - f32(0.5) / s2).astype(np.float32)


def loss_vertex(pred, targ, listed, w_inside, sigma):
    """Expected [2] output of the fused loss: pred / targ [B,H,W,3] float32 (each pixel's own class), listed [B,H,W].
    Returns dict(out0, out1 (float32), S (exact term sum), count, n_terms, bound (double-accumulation bound), boundary
    (terms with |diff| == 1 / sigma^2), tiny (terms below 2^-30), terms)."""
    s2 = f32(sigma) * f32(sigma)
    terms = sl1_terms(pred[listed], targ[listed], w_inside, sigma)
    diff = np.abs(f32(w_inside) * (pred[listed] - targ[listed]))
    count = int(listed.sum())
    n_terms = terms.size
    S = exact_sum(terms)
    W = Fraction(3) * Fraction(float(f32(w_inside))) * count
    D = Fraction(float(W) + 1e-10)                           # tw + 1e-10 in double; tw is exact
    assert float(W) == W
    # any order of double additions over the terms, the per-thread and per-warp partials and the last CTA's pass
    N = n_terms + LOSS_BLOCKS * (LOSS_THREADS + LOSS_THREADS // 32 + 1)
    abs_sum = exact_sum(np.abs(terms))
    delta = Fraction(N) * Fraction(2) ** -53 * abs_sum * Fraction(1 + 2 ** -20)
    lo = (S - delta) / D * (1 - Fraction(2) ** -53)
    hi = (S + delta) / D * (1 + Fraction(2) ** -53)
    lo_d = np.nextafter(float(lo), -math.inf)
    hi_d = np.nextafter(float(hi), math.inf)
    out0 = _f32_of(S / D)
    if not (_f32_of(lo_d) == out0 == _f32_of(hi_d)):
        raise Straddle(f"loss interval [{lo_d!r}, {hi_d!r}] straddles an fp32 rounding boundary")
    return dict(out0=out0, out1=np.float32(float(W)), S=S, count=count, n_terms=n_terms, bound=float(delta),
                boundary=int((diff == f32(1) / s2).sum()), tiny=int((terms < 2.0 ** -30).sum()), terms=terms)


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------
def _units(sigma):
    """Grid of the low-resolution vertex channels: predictions land on unit / 256, fine enough to hold f32(1 / sigma^2)
    (a multiple of 2^-25 at sigma = 2.5) and coarse enough for |pred| < 2^24 unit / 256."""
    return 2.0 ** -15 if f32(1) / (f32(sigma) * f32(sigma)) == 1 else 2.0 ** -17


def loss_problem(B, H, W, C, coord, sigma, gen, w_inside=1.0):
    """Operands of the fused loss (numpy / CPU torch).  The vertex channels of lowres are multiples of `unit` in
    [-1/4, 1/4], the biases multiples of unit / 256 in [-1/8, 1/8], except:
    - zero blocks: 3 x 3 low-resolution cells whose vertex channels are 0, so the 16 x 16 pixels they cover predict exactly
      the bias; the planted classes' bias of channel k_p is +-f32(1 / sigma^2) / w, and their target there is 0 (2-D: the
      dy channel on the centre's row; 3-D: a zero extent on axis 1), so |w (pred - target)| == 1 / sigma^2: the branch
      boundary of sl1_term;
    - a tiny band: the first four low-resolution rows hold multiples of unit in [-8 unit, 8 unit], the log-z biases are as
      small, and every third class has z = 1 (2-D: log-z target 0); in 3-D the vertmap there makes the targets equal the
      predictions up to rounding, so those terms are tiny.
    Labels: -1, background, values C and C + 1, labelled classes that are not listed (z = 0, NaN or negative), and
    foreground; the last pixel of the batch is a listed foreground pixel.  Centres are multiples of 2^-12, z from
    LOGZ_TABLE (2-D).  3-D extents are float32 values in [0.03, 0.3] (zero on the planted axes) and the vertmap
    float32 values in [-0.15, 0.15], so every float32 operation of coord_scale / coord_target rounds."""
    h, w = H // 8, W // 8
    unit = _units(sigma)
    rng = np.random.default_rng(int(torch.randint(0, 2 ** 31, (1,), generator=gen)))
    lowres = R.dyadic((B, h, w, 4 * C), -1, 1, 0.125, gen)
    lowres[..., C:] = R.dyadic((B, h, w, 3 * C), -0.25, 0.25, unit, gen)
    lowres[:, :4, :, C:] = R.dyadic((B, 4, w, 3 * C), -8 * unit, 8 * unit, unit, gen)
    bias_v = R.dyadic((3 * C,), -0.125, 0.125, unit / 256, gen)
    bias_v[2::3] = R.dyadic((C,), -8 * unit, 8 * unit, unit / 256, gen)
    d = float(f32(1) / (f32(sigma) * f32(sigma))) / float(f32(w_inside))
    planted = list(range(1, C, 3)) if C > 2 else [1]
    if d / (unit / 256) != round(d / (unit / 256)):
        planted = []                                          # 1 / (sigma^2 w) is off the grid (w_inside = 10): no boundary
    for c in planted:
        bias_v[3 * c + 1] = d if c % 2 else -d
    # zero blocks on a regular lattice, rows of cells 6.., every ninth cell
    blocks = [(i, j) for i in range(6, h - 3, 9) for j in range(1, w - 3, 9)]
    for (i, j) in blocks:
        lowres[:, i:i + 3, j:j + 3, C:] = 0
    # labels
    r = rng.integers(0, 100, (B, H, W))
    fg = rng.integers(1, C, (B, H, W)) if C > 2 else np.ones((B, H, W), np.int64)
    label = np.where(r < 8, -1, np.where(r < 10, C + (r - 8), np.where(r < 30, 0, fg)))
    centers = np.zeros((B, C, 3), np.float32)
    centers[..., 0] = rng.integers(-64 * 4096, (W + 64) * 4096, (B, C)) / 4096
    centers[..., 1] = rng.integers(-64 * 4096, (H + 64) * 4096, (B, C)) / 4096
    centers[..., 2] = LOGZ_TABLE[rng.integers(0, LOGZ_TABLE.size, (B, C))]
    centers[:, 3::3, 2] = 1.0                                 # log z = 0: tiny log-z terms in the tiny band
    centers[:, 0] = (10.0, 10.0, 1.0)                         # background slot: never read
    if C > 2:
        centers[0, 2, 2] = 0.0                                # labelled, not listed
        centers[0, 3, 2] = np.nan
        centers[B - 1, 5, 2] = -1.0
    else:
        centers[0, 1, 2] = 0.0
    unlisted = ~(centers[..., 2] > 0)
    # planted pixels: in each zero block, a row of a planted class with dy == 0 (2-D: the centre sits on that row)
    for n, (i, j) in enumerate(blocks if planted else []):
        b, c = n % B, planted[n % len(planted)]
        if unlisted[b, c]:
            continue
        y0, x0 = 8 * i + 4, 8 * j + 4
        label[b, y0:y0 + 16, x0:x0 + 16] = c
        if not coord:
            centers[b, c, 1] = y0 + 5
            label[b, y0 + 5, x0:x0 + 16] = c
    # the last pixel: listed foreground
    last_c = next(c for c in range(C - 1, 0, -1) if not unlisted[B - 1, c])
    label[B - 1, H - 1, W - 1] = last_c
    P = dict(B=B, H=H, W=W, C=C, coord=coord, sigma=sigma, w_inside=w_inside, unit=unit, lowres=lowres, bias_v=bias_v,
             label=label.astype(np.int32), centers=centers, blocks=blocks, planted=planted)
    if coord:
        # object extents of YCB-like size: a = 1 / span and b = -vmin / span round, and so does a v, so a contraction of
        # coord_target into an FMA or another order of _scale_vertmap's float32 operations changes targets
        ext = rng.uniform(0.03, 0.3, (C, 3)).astype(np.float32)
        ext[planted, 1] = 0.0                                 # a = b = 0: target 0 on axis 1
        P["extents"] = ext
        vm = rng.uniform(-0.15, 0.15, (B, H, W, 3)).astype(np.float32)
        # tiny band: v = (pred - b) / a rounded, so the target a v + b equals the prediction up to rounding
        listed, cls, _ = _listed(label, centers[..., 2], C)
        pv, _ = own_vertex_values(lowres, bias_v, cls, C, unit)
        ab = R.coord_scale(torch.as_tensor(ext)).numpy().astype(np.float64)[cls]          # [B,H,W,3,2]
        band = np.zeros((B, H, W, 1), bool)
        band[:, :28] = True
        a = ab[..., 0]
        v_tiny = ((pv.astype(np.float64) - ab[..., 1]) / np.where(a > 0, a, 1)).astype(np.float32)
        vm = np.where(band & (a > 0), v_tiny, vm)
        P["vertmap"] = vm.astype(np.float32)
    return P


def reference(P, label=None):
    """Targets, own-class predictions and the expected loss of problem P (optionally with another label map)."""
    label = P["label"] if label is None else label
    if P["coord"]:
        listed, cls, t = targets_3d(label, P["vertmap"], P["centers"], P["extents"])
    else:
        listed, cls, t = targets_2d(label, P["centers"])
    pv, budget = own_vertex_values(P["lowres"], P["bias_v"], cls, P["C"], P["unit"])
    L = loss_vertex(pv, t, listed, P["w_inside"], P["sigma"])
    L.update(listed=listed, cls=cls, t=t, pv=pv, budget=budget)
    return L


def loss_plan(npix):
    """Grid-stride coverage of the fused losses: kLossBlocks x 256 threads."""
    sweep = LOSS_BLOCKS * LOSS_THREADS
    return dict(npix=npix, sweep=sweep, sweeps=npix / sweep, tail=npix % sweep)


# ---------------------------------------------------------------------------------------------------------------------
# pose blob and meta packing (k_pack_pose_meta)
# ---------------------------------------------------------------------------------------------------------------------
def pack_pose_meta(poses, cls, intrinsics, im_scale, flip_x):
    """pose_blob [B*I,13] (listed rows in order, zero rows after), num_rows and meta [B,48] in float64 rounded to float32.
    The quaternion is the float64 one of scipy (w, x, y, z with w >= 0); meta's K = float32 intrinsics times the float32
    im_scale, K[2][2] = 1, and its inverse by cofactors: on intrinsics with few significant bits every product and sum is
    exact in double (so a contraction cannot change it) and each entry is one correctly rounded division."""
    from scipy.spatial.transform import Rotation
    poses, cls = np.asarray(poses, np.float32), np.asarray(cls)
    B, I = cls.shape
    blob = np.zeros((B * I, 13), np.float32)
    n = 0
    for k in range(B * I):
        b, i = divmod(k, I)
        if cls[b, i] < 0:
            continue
        q = Rotation.from_matrix(poses[b, i, :, :3].astype(np.float64)).as_quat()     # x, y, z, w
        q = np.r_[q[3], q[:3]]
        blob[n] = [b, cls[b, i], 0, 0, 0, 0, *(q if q[0] >= 0 else -q), *poses[b, i, :, 3]]
        n += 1
    meta = np.zeros((B, 48), np.float32)
    for b in range(B):
        K = np.asarray(intrinsics[b], np.float32).astype(np.float64).ravel() * np.float64(np.float32(im_scale))
        K[8] = 1.0
        c = [K[4] * K[8] - K[5] * K[7], K[5] * K[6] - K[3] * K[8], K[3] * K[7] - K[4] * K[6]]
        det = K[0] * c[0] + K[1] * c[1] + K[2] * c[2]
        cof = [c[0], K[2] * K[7] - K[1] * K[8], K[1] * K[5] - K[2] * K[4],
               c[1], K[0] * K[8] - K[2] * K[6], K[2] * K[3] - K[0] * K[5],
               c[2], K[1] * K[6] - K[0] * K[7], K[0] * K[4] - K[1] * K[3]]
        meta[b, :9] = K
        meta[b, 9:18] = [x / det for x in cof]
        if flip_x:
            meta[b, [0, 9, 11]] *= -1
    return blob, n, meta
