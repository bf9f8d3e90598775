"""The references of tests/pose_bwd_ref.py checked without a GPU: against the C oracle, against float64 autograd of the
reference formula, against fp32 torch computations done in another order, and against exact rational arithmetic."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import oracle
from tests import pose_bwd_ref as R
from tests.train_ref import ad_loss_torch, quat_rot


def test_quat_jacobians_match_autograd():
    q = torch.randn(16, 4, dtype=torch.float64)
    J = R.quat_jacobians(q)
    for n in range(16):
        jac = torch.autograd.functional.jacobian(quat_rot, q[n])         # [3,3,4]
        assert torch.equal(jac.permute(2, 0, 1), J[n])


def _ad_small(seed, N=32, C=4, P=256):
    g = torch.Generator().manual_seed(seed)
    pb = R.ad_problem(N, C, P, g, zero_frac=0.3)
    ref = R.average_distance(pb["pred"], pb["target"], pb["weight"], pb["points"], pb["symmetry"], pb["margin"], units=pb["units"])
    return pb, ref


def test_average_distance_ref_equals_oracle_on_dyadic_operands():
    """The C oracle (fp32 arithmetic, double sums) equals the float64 reference bit for bit on dyadic operands."""
    for seed in (1, 2):
        pb, ref = _ad_small(seed)
        print(f"seed {seed}: ties {ref['ties']}, hinge ties {ref['hinge_ties']}, budgets row grad {ref['budget_row_grad']:.0f} "
              f"row loss {ref['budget_row_loss']:.0f} batch {ref['budget_batch_loss']:.0f}")
        assert ref["ties"] > 0 and ref["hinge_ties"] > 0 and ref["sym_rows"] > 0
        loss, diff = oracle.average_distance_loss(*(pb[k].numpy() for k in ("pred", "target", "weight", "points", "symmetry")), pb["margin"])
        assert loss[0] == np.float32(ref["loss"].item())
        assert np.array_equal(diff, ref["diff"].float().numpy())


def _ad_loss_fixed(pred, target, cls, points, match, margin):
    """Averagedistance with each point's gt partner fixed (match): the symmetric rows' loss with the argmin held constant,
    differentiable in pred (same hinge as train_ref.ad_loss_torch: d == margin takes the d - margin branch)."""
    N, D = pred.shape
    P = points.shape[1]
    loss = pred.new_zeros(())
    for n in range(N):
        c = int(cls[n])
        if c < 0:
            continue
        Ru, Rg = quat_rot(pred[n, 4 * c:4 * c + 4]), quat_rot(target[n, 4 * c:4 * c + 4])
        a, b = points[c] @ Ru.t(), (points[c] @ Rg.t())[match[n]]
        d = (a - b).pow(2).sum(1)
        loss = loss + torch.where(d < margin, torch.zeros_like(d), d - margin).sum() / (2.0 * N * P)
    return loss


def test_average_distance_ref_equals_float64_autograd():
    """Float64 autograd of train_ref.ad_loss_torch (non-symmetric rows) and of the fixed-argmin variant (all rows) gives the
    reference's gradient exactly; loss equal too."""
    pb, ref = _ad_small(3, N=16, P=128)
    pred = pb["pred"].double().requires_grad_(True)
    sym = pb["symmetry"][ref["cls"].clamp(min=0)] > 0
    wns = pb["weight"].double() * (~sym | (ref["cls"] < 0))[:, None]
    ad_loss_torch(pred, pb["target"].double(), wns, pb["points"].double(), pb["margin"]).backward()
    nonsym = (ref["cls"] >= 0) & ~sym
    assert int(nonsym.sum()) > 0
    # ad_loss_torch normalises by the same N P: rows without weight contribute nothing
    assert torch.equal(pred.grad[nonsym], ref["diff"][nonsym])
    pred.grad = None
    loss = _ad_loss_fixed(pred, pb["target"].double(), ref["cls"], pb["points"].double(), ref["match"].clamp(min=0), pb["margin"])
    loss.backward()
    assert torch.equal(pred.grad, ref["diff"])
    assert loss.item() == ref["loss"].item()


def test_average_distance_budget_fires():
    g = torch.Generator().manual_seed(4)
    pb = R.ad_problem(8, 4, 64, g)
    with pytest.raises(R.BudgetExceeded):
        R.average_distance(pb["pred"] * 2 ** 11, pb["target"], pb["weight"], pb["points"], pb["symmetry"], pb["margin"], units=pb["units"])


def test_average_distance_bound_covers_fp32_torch():
    """On unit quaternions the derived bound covers an fp32 torch evaluation of the same formula (another summation order)."""
    from posecnn_b200 import synth
    pred, targ, wt = (torch.from_numpy(a) for a in synth.make_pose_batch(24, 22, seed=5))
    pts, sym = torch.from_numpy(synth.make_model_points(22, 300)), torch.from_numpy(synth.LOV_SYMMETRY)
    ref = R.average_distance(pred, targ, wt, pts, sym, 0.01)
    b = R.ad_bound(pred, targ, wt, pts, sym, 0.01, ref)
    loss32, diff32 = oracle.average_distance_loss(pred.numpy(), targ.numpy(), wt.numpy(), pts.numpy(), sym.numpy(), 0.01)
    assert ((torch.from_numpy(diff32).double() - ref["diff"]).abs() <= b["grad"]).all()
    assert abs(float(loss32[0]) - ref["loss"].item()) <= b["loss"] + 2 ** -24 * ref["loss"].item()


def test_pose_chain_bound_covers_fp32_torch():
    """The float64 pose-chain reference and its bound cover an fp32 torch evaluation (torch.rsqrt, different sum order)."""
    g = torch.Generator().manual_seed(6)
    P = R.pose_chain_problem(64, 22, g)
    for up in (1.0, 2.0 ** 24):
        d, err, clamped = R.pose_chain(P["g"], P["tanh"], P["w"], up)
        assert bool(clamped[0]) and bool(clamped[1]) and not bool(clamped[2:].any())
        u = P["tanh"] * P["w"]
        gg = up * P["g"]
        su = (u * u).sum(1, keepdim=True)
        inv = torch.rsqrt(su.clamp(min=1e-12))
        du = torch.where(su < 1e-12, gg * inv, (gg - u * inv * ((u * gg).sum(1, keepdim=True) * inv)) * inv)
        d32 = du * P["w"] * (1 - P["tanh"] * P["tanh"])
        assert ((d32.double() - d).abs() <= err).all()
        assert float((err / d.abs().clamp(min=1e-30))[d != 0].median()) < 1e-5      # not vacuous (it grows under cancellation)


def test_f16_saturation():
    x = torch.tensor([float("nan"), float("inf"), -float("inf"), 70000.0, -65520.0, 65519.0, 1e-7, -6e-8])
    y = R.f16_sat(x)
    assert torch.isnan(y[0]) and y[1:6].tolist() == [65504.0, -65504.0, 65504.0, -65504.0, 65504.0]
    assert y[6].item() == float(torch.tensor(1e-7).half()) and y[7].item() == float(torch.tensor(-6e-8).half())


def test_roundf_half_away_from_zero():
    x = torch.tensor([-2.5, -1.5, -0.5, 0.5, 1.5, 2.5, 0.49999997, -0.49999997])
    assert R.roundf(x).tolist() == [-3, -2, -1, 1, 2, 3, 0, 0]


@pytest.mark.parametrize("scale,hw", [(1 / 16, (30, 40)), (1 / 8, (60, 80))], ids=["conv5_3", "conv4_3"])
def test_roi_scatter_equals_oracle(scale, hw):
    """The Python acceptance rule and scatter equal oracle.roi_pool_grad (the reference's per-element gather over every ROI)
    on a channel-reduced copy of the training-shape problem, with the oracle's own argmax."""
    g = torch.Generator().manual_seed(7)
    B, Cc = 2, 8
    rois = R.train_rois(g)
    H, W = hw
    feat = torch.randint(0, 4, (B, H, W, Cc), generator=g).float()
    valid = (rois[:, 0] >= 0) & (rois[:, 0] < B)
    arg = np.full((rois.shape[0], 7, 7, Cc), -1, np.int32)
    arg[valid.numpy()] = oracle.roi_pool(feat.numpy(), rois[valid].numpy(), 7, 7, scale)[1]
    dpool = R.dyadic((rois.shape[0], 7, 7, Cc), -8, 8, 1.0, g) * 2.0 ** -6
    want = oracle.roi_pool_grad(feat.numpy(), rois.numpy(), arg, dpool.numpy(), 7, 7, scale)
    got, budget, accepted = R.roi_pool_grad((B, H, W, Cc), rois, torch.from_numpy(arg), dpool, scale, 2.0 ** -6)
    print(f"{rois.shape[0]} rows, {accepted} accepted (bin, channel) pairs, budget {budget:.0f}")
    assert accepted > 0
    assert np.array_equal(got.float().numpy(), want)
    # the malformed boxes are pooled forward but rejected backward
    geo = R.roi_geometry(rois, scale)
    bad = (geo["rew"] < geo["rsw"]) & valid
    assert int(bad.sum()) >= 1 and bool((torch.from_numpy(arg)[bad] >= 0).all())
    ok = R.roi_accepts(geo, torch.from_numpy(arg), H, W, Cc)
    assert not bool(ok[bad].any())


def _fma_exact(a, b, c):
    """fp32 fma by rational arithmetic: the nearest fp32 to a b + c, ties to even."""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = np.float32(float(x))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    best = min(abs(Fraction(float(v)) - x) for v in cands)
    near = [v for v in cands if abs(Fraction(float(v)) - x) == best]
    return near[0] if len(near) == 1 else next(v for v in near if int(np.array(v).view(np.uint32)) % 2 == 0)


def test_fmaf_emulation_is_exact():
    g = torch.Generator().manual_seed(8)
    a = torch.randn(3000, generator=g) * torch.exp2(torch.randint(-20, 20, (3000,), generator=g).float())
    b = torch.randn(3000, generator=g)
    c = torch.randn(3000, generator=g) * torch.exp2(torch.randint(-20, 20, (3000,), generator=g).float())
    # float64 sums that fall exactly on an fp32 midpoint with a residual beyond float64: (1 +- 2^-23) 2^-25 (1 -+ 2^-23) + c
    e = 2.0 ** -23
    planted = [(1 + e, -(1 - e) * 2.0 ** -25, 1.0), (1 + e, (1 - e) * 2.0 ** -25, 1 - 2.0 ** -24), (0.001, 0.9, 1e-4),
               (3.0, 1 / 3, -1.0)]
    pa, pb, pc = (torch.tensor([p[k] for p in planted], dtype=torch.float32) for k in range(3))
    a, b, c = torch.cat([a, pa]), torch.cat([b, pb]), torch.cat([c, pc])
    got = R.fmaf(a, b, c)
    want = torch.tensor([_fma_exact(*v) for v in zip(a.numpy(), b.numpy(), c.numpy())])
    assert torch.equal(got, want)
    naive = (a.double() * b.double() + c.double()).float()
    assert not torch.equal(naive[-4:], want[-4:])          # the planted midpoints defeat a plain double rounding


@pytest.mark.parametrize("kind", ["bf16", "fp16"])
def test_sgd_dyadic_steps_are_exact(kind):
    """Three carried steps of the dyadic momentum update: the fp32 emulation equals the unrounded float64 update, and the
    planted ties are ties of the 16-bit copy."""
    g = torch.Generator().manual_seed(9)
    H = R.SGD_DYADIC
    w = R.dyadic((4096,), -1, 1, 2.0 ** -11, g)
    acc = R.dyadic((4096,), -1, 1, 2.0 ** -4, g)
    for step in range(3):
        grad, tie = R.sgd_step_operands(w, acc, g, kind)
        w64, a64 = R.sgd_f64(w, acc, grad, **H)
        w, acc = R.sgd_fp32(w, acc, grad, **H)
        assert torch.equal(w.double(), w64) and torch.equal(acc.double(), a64)
        low = w[tie].view(torch.int32) & (0xFFFF if kind == "bf16" else 0x1FFF)
        assert int(tie.sum()) > 100 and bool((low == (0x8000 if kind == "bf16" else 0x1000)).all())


def test_sgd_budget_fires():
    g = torch.Generator().manual_seed(10)
    w = R.dyadic((256,), -1, 1, 2.0 ** -20, g)
    with pytest.raises(R.BudgetExceeded):
        R.sgd_step_operands(w, torch.zeros(256), g, "bf16")


def test_plans():
    assert R.ad_plan(1024, 2048) == dict(grid=1024, threads=256, points_per_thread=8, batch_items_per_thread=4)
    assert R.pose_chain_plan(1152, 168, 256) == dict(grid=144, rows_per_cta=8, last_cta_rows=8, cols_per_lane=6, out_per_lane=8)
    assert R.pose_chain_plan(7, 24, 128)["last_cta_rows"] == 7
    p = R.ew_plan(102760448 + 3)
    assert p["grid"] == 1056 and p["ragged"] and p["items_per_thread"] == 381
