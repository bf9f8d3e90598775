"""The pose-regression backward of the training step at training shapes: Averagedistance and its gradient, the pose chain
(l2_normalize o x weight o tanh adjoint), RoiPool's argmax and gradient, and the momentum update with the trainer's copies.

Averagedistance, RoiPool's gradient and the momentum update run on dyadic operands (tests/pose_bwd_ref.py), where every fp32
operation of the kernel is exact in any order (checked bit budgets): their outputs must equal the float64 references bit for
bit.  The pose chain goes through rsqrtf and is held to a derived error interval, the realistic Averagedistance case to a
derived bound, the realistic momentum update to an exact fp32 emulation of fmaf.  Each test prints the launch plan it covered
and asserts that coverage."""
import math

import numpy as np
import pytest
import torch

from tests import pose_bwd_ref as R

pytestmark = pytest.mark.gpu


def assert_same(got, want, what):
    """Equal values (+0 == -0), NaN where the other is NaN."""
    nan = torch.isnan(got)
    assert torch.equal(nan, torch.isnan(want)), f"{what}: NaN positions differ"
    bad = (got != want) & ~nan
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} values differ; first at {bad.nonzero()[0].tolist()}: "
                                 f"{got[tuple(bad.nonzero()[0])].item()} != {want[tuple(bad.nonzero()[0])].item()}")


# ---------------------------------------------------------------------------------------------------------------------
# 1. Averagedistance, exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,P", [(1024, 2048), (64, 32), (8, 1)])
def test_average_distance_exact(cuda, N, P):
    """loss and bottom_diff bit for bit against float64 on dyadic operands; 1024 rows of 2048 points is the training step's
    scale (1024 CTAs for 132 SMs, so the last-CTA batch reduction runs after many completions).  Rows without a weighted class
    give zero rows; symmetric rows include equidistant distinct gt points (first minimum wins) and points at dist == margin
    (no loss, but gradient).  A second launch is bit-identical (the completion counter is reset), and the gradient op is exact
    for a power-of-two upstream."""
    from posecnn_b200.average_distance_loss import average_distance_loss_op as op
    C = 4
    plan = R.ad_plan(N, P)
    print(f"N={N} P={P} D={4 * C}: {plan['grid']} CTAs x {plan['threads']} threads, {plan['points_per_thread']} points per thread, "
          f"batch loss {plan['batch_items_per_thread']} rows per thread of the last CTA")
    assert plan["grid"] == N and plan["points_per_thread"] == math.ceil(P / 256)
    g = torch.Generator().manual_seed(N + P)
    pb = R.ad_problem(N, C, P, g, zero_frac=0.85 if N * P >= 1 << 20 else 0.3)
    T = {k: pb[k].to(cuda) for k in ("pred", "target", "weight", "points", "symmetry")}
    ref = R.average_distance(T["pred"], T["target"], T["weight"], T["points"], T["symmetry"], pb["margin"], units=pb["units"])
    print(f"budgets: term {ref['budget_term']:.0f}, row gradient {ref['budget_row_grad']:.0f}, row loss {ref['budget_row_loss']:.0f}, "
          f"batch loss {ref['budget_batch_loss']:.0f} (limit 2^24 = {R.LIMIT}); symmetric rows {ref['sym_rows']}, equidistant "
          f"distinct minima {ref['ties']}, points at dist == margin {ref['hinge_ties']}")
    cls = ref["cls"]
    assert bool((cls < 0).any()) and bool((cls >= 0).any())
    assert ref["sym_rows"] > 0
    if N * P >= 1 << 20:
        assert ref["ties"] > 0 and ref["hinge_ties"] > 0
    args = (T["pred"], T["target"], T["weight"], T["points"], T["symmetry"], pb["margin"])
    loss, diff = op.average_distance_loss(*args)
    loss2, diff2 = op.average_distance_loss(*args)
    torch.cuda.synchronize()
    assert_same(loss[0], ref["loss"].float(), "loss")
    assert_same(diff, ref["diff"].float(), "bottom_diff")
    assert bool((diff[cls < 0] == 0).all())
    assert torch.equal(loss.view(torch.int32), loss2.view(torch.int32)) and torch.equal(diff.view(torch.int32), diff2.view(torch.int32))
    up = torch.tensor([2.0 ** -3], device=cuda)
    assert_same(op.average_distance_loss_grad(diff, up), (ref["diff"] * 2.0 ** -3).float(), "bottom_diff x upstream")


# ---------------------------------------------------------------------------------------------------------------------
# 2. Averagedistance, realistic
# ---------------------------------------------------------------------------------------------------------------------
def test_average_distance_realistic_bound(cuda):
    """The bench's problem (unit quaternions, 2620 model points, margin 0.01, 1152 rows, C = 22, LOV symmetry) within the
    derived error bound of the float64 reference; ambiguous points (hinge or symmetric argmin within the error) widen it."""
    from posecnn_b200 import synth
    from posecnn_b200.average_distance_loss import average_distance_loss_op as op
    N, C, P = 1152, 22, 2620
    plan = R.ad_plan(N, P)
    print(f"N={N} P={P} D={4 * C}: {plan['grid']} CTAs, {plan['points_per_thread']} points per thread")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    pred, targ, wt = (T(a) for a in synth.make_pose_batch(N, C, seed=9))
    pts, sym = T(synth.make_model_points(C, P)), T(synth.LOV_SYMMETRY)
    ref = R.average_distance(pred, targ, wt, pts, sym, 0.01, chunk=16)
    b = R.ad_bound(pred, targ, wt, pts, sym, 0.01, ref, chunk=16)
    loss, diff = op.average_distance_loss(pred, targ, wt, pts, sym, 0.01)
    err = (diff.double() - ref["diff"]).abs()
    nz = ref["diff"] != 0
    print(f"symmetric rows {ref['sym_rows']}, ambiguous points {b['ambiguous']}; max |err| / bound {float((err / b['grad'].clamp(min=1e-300))[nz].max()):.3g}; "
          f"loss err {abs(loss.item() - ref['loss'].item()):.3g} bound {b['loss']:.3g}")
    assert ref["sym_rows"] > 0
    assert bool((err <= b["grad"]).all())
    assert abs(loss.item() - ref["loss"].item()) <= b["loss"]


# ---------------------------------------------------------------------------------------------------------------------
# 3. the pose chain
# ---------------------------------------------------------------------------------------------------------------------
def _chain(P, upstream, cuda, ld):
    from posecnn_b200 import pose_head
    N = P["g"].shape[0]
    g, t, w = (P[k].to(cuda).contiguous() for k in ("g", "tanh", "w"))
    out = torch.full((N, ld), 7.0, dtype=torch.float16, device=cuda)          # padding columns must be written as 0
    pose_head.pose_chain_bwd(g, t, w, upstream, out)
    torch.cuda.synchronize()
    return out.cpu()


def _check_chain(out, P, upstream, what):
    D = P["g"].shape[1]
    d, err, clamped = R.pose_chain(P["g"], P["tanh"], P["w"], upstream)
    got = out[:, :D].float()
    assert bool((out[:, D:].view(torch.int16) == 0).all()), f"{what}: padding columns not zero"
    fin = torch.isfinite(d)
    lo, hi = R.f16_sat(d - err).float(), R.f16_sat(d + err).float()
    assert bool(((got >= lo) & (got <= hi))[fin].all()), f"{what}: outside the derived interval"
    assert_same(got[~fin], R.f16_sat(d[~fin]).float(), f"{what}: non-finite")
    live = P["w"] != 0
    exact = float((got == R.f16_sat(d).float())[live].double().mean())
    return exact, clamped


@pytest.mark.parametrize("D", [8, 24, 88, 168])
@pytest.mark.parametrize("rows", [1, 7, 1151, 1152])
def test_pose_chain(cuda, rows, D):
    """pcnn_pose_chain_bwd inside the derived fp32 interval after fp16 rounding, >= 99 % of the weighted elements equal to
    fp16(reference), padding columns 0; D = 168 is C = 42 with its 256-column stride.  Upstream 1 and 2^24.  1152 rows is the
    step's largest ROI count; 7 and 1151 leave the last CTA partly idle."""
    C = D // 4
    P = R.pose_chain_problem(rows, C, torch.Generator().manual_seed(rows * 1000 + D))
    ld = P["ld"]
    plan = R.pose_chain_plan(rows, D, ld)
    print(f"rows={rows} D={D} ld={ld}: {plan['grid']} CTAs x {plan['rows_per_cta']} rows, last CTA {plan['last_cta_rows']} rows, "
          f"{plan['cols_per_lane']} columns per lane, {plan['out_per_lane']} outputs per lane")
    assert ld == (128 if D <= 128 else 256) and plan["cols_per_lane"] == math.ceil(D / 32)
    if rows % 8:
        assert plan["last_cta_rows"] < 8
    for up in (1.0, 2.0 ** 24):
        exact, clamped = _check_chain(_chain(P, up, cuda, ld), P, up, f"upstream {up}")
        print(f"  upstream {up:g}: {exact:.4%} of weighted elements equal fp16(ref); clamped rows {int(clamped.sum())}")
        assert exact >= 0.99
        if rows > 2:
            assert int(clamped.sum()) == 2


def test_pose_chain_edges(cuda):
    """Clamped rows (zero weights; tiny tanh values with sum u^2 < 1e-12: du = g / 1e-6), saturation at +-65504 under
    S = 2^24, fp16 subnormal outputs, +-inf inputs (-> +-65504) and NaN (-> NaN)."""
    N, C = 24, 6
    P = R.pose_chain_problem(N, C, torch.Generator().manual_seed(77))
    cols = (P["w"][1] != 0).nonzero().flatten()
    P["g"][1, cols[:3]] = torch.tensor([float("inf"), -float("inf"), float("nan")])
    P["g"][2:8] *= 1e3                                                         # overflow at S = 2^24
    P["g"][8:16] *= 1e-2                                                       # subnormal at S = 1
    for up in (2.0 ** 24, 1.0):
        out = _chain(P, up, cuda, P["ld"])
        _check_chain(out, P, up, f"upstream {up}")
        o = out.float()
        sat, sub = int((o.abs() == 65504).sum()), int(((o != 0) & (o.abs() < 2.0 ** -14)).sum())
        print(f"upstream {up:g}: {sat} saturated, {sub} subnormal, NaN {int(torch.isnan(o).sum())}")
        assert torch.isnan(o[1, cols[2]]) and o[1, cols[0]].item() == 65504.0 and o[1, cols[1]].item() == -65504.0
        assert (sat > 10) if up > 1 else (sub > 10)


def test_pose_step_beyond_32_classes(cuda):
    """C = 42 (D = 168 > 128): the step's pose chain uses a 256-column dpre stride, fc8's padded weight rows get zero
    gradient and the gradients are finite."""
    from posecnn_b200.train import Trainer
    from tests.train_ref import make_inputs, make_net, synthetic_pose_targets
    C = 42
    net = make_net(cuda, C=C)
    args, _, _ = make_inputs(cuda, C=C)
    tr = Trainer(net)
    A = tr.forward(*args)
    synthetic_pose_targets(A, args[6] * 10, args[7], tr.margin)      # model points x 10: distances well above the margin
    grads = tr.backward(A, args[1], args[2])
    torch.cuda.synchronize()
    print(f"rows {A['rows']}, fc8 master {tuple(tr.master['fc8/w'].shape)}, loss scale {tr.pose_loss_scale:g}")
    assert A["pose_diff"].abs().max() > 0
    assert tr.master["fc8/w"].shape[0] == 256 and grads["fc8/w"].shape == tr.master["fc8/w"].shape
    assert bool((grads["fc8/w"][4 * C:] == 0).all()) and bool(grads["fc8/w"][:4 * C].abs().sum() > 0)
    assert all(bool(torch.isfinite(v).all()) for v in grads.values())


# ---------------------------------------------------------------------------------------------------------------------
# 4. RoiPool at training shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale,hw", [(1 / 16, (30, 40)), (1 / 8, (60, 80))], ids=["conv5_3", "conv4_3"])
def test_roi_pool_argmax_and_grad_exact(cuda, scale, hw):
    """The s4 forward's argmax equals the C oracle's on small-integer bf16 features (ties everywhere), and the gradient
    scatter equals a float64 scatter with the reference's acceptance tests bit for bit, whatever the atomic order."""
    from oracle import oracle
    from posecnn_b200.roi_pooling_layer import roi_pooling_op as rop
    g = torch.Generator().manual_seed(int(1 / scale))
    B, Cc = 2, 512
    H, W = hw
    rois = R.train_rois(g)
    N = rois.shape[0]
    feat = torch.randint(0, 4, (B, H, W, Cc), generator=g).to(torch.bfloat16)
    plan = R.roi_bwd_plan(N, Cc)
    geo = R.roi_geometry(rois, scale)
    valid = (geo["b"] >= 0) & (geo["b"] < B)
    xs = rois[:, 2:6] * scale
    halves = int((xs - xs.floor() == 0.5).any(1).sum())
    malformed = int(((geo["rew"] < geo["rsw"]) & valid).sum())
    print(f"{H}x{W}x{Cc}, {N} rows ({int((~valid).sum())} foreign batch, {malformed} malformed, {halves} with a .5 corner): bwd grid "
          f"{plan['grid']} CTAs, {plan['items_per_thread']} items per thread")
    assert N >= 1000 and int((~valid).sum()) >= 3 and malformed >= 1 and halves >= 100 and plan["items_per_thread"] >= 2
    d_feat, d_rois = feat.to(cuda), rois.to(cuda)
    _, arg = rop.roi_pool(d_feat, d_rois, 7, 7, scale, 0)
    arg = arg.cpu()
    want = oracle.roi_pool(feat.float().numpy(), rois[valid].numpy(), 7, 7, scale)[1]
    assert np.array_equal(arg[valid].numpy(), want)
    assert bool((arg[~valid] == -1).all())
    unit = 2.0 ** -6
    dpool = R.dyadic((N, 7, 7, Cc), -8, 8, 1.0, g) * unit
    got = rop.roi_pool_grad(d_feat, d_rois, arg.to(cuda), dpool.to(cuda), 7, 7, scale, 0).cpu()
    ref, budget, accepted = R.roi_pool_grad((B, H, W, Cc), rois, arg, dpool, scale, unit)
    print(f"accepted (bin, channel) pairs {accepted} of {int((arg >= 0).sum())} with an argmax; per-element budget {budget:.0f}")
    assert accepted < int((arg[valid] >= 0).sum())                  # the acceptance tests reject some pairs
    assert_same(got, ref.float(), "roi_pool_grad")


# ---------------------------------------------------------------------------------------------------------------------
# 5. SGD with momentum and the trainer's update
# ---------------------------------------------------------------------------------------------------------------------
def _sgd(w, acc, grad, H, kind):
    from posecnn_b200._lib import check, lib, ptr, stream
    copy = torch.empty(w.shape, dtype=torch.float16 if kind == "fp16" else torch.bfloat16, device=w.device)
    check(lib().pcnn_sgd_momentum(ptr(w), ptr(acc), ptr(grad), w.numel(), H["lr"], H["mu"], H["wd"], H["gscale"], ptr(copy),
                                  int(kind == "fp16"), stream()))
    torch.cuda.synchronize()
    return copy


def _copy_ref(w, kind):
    return R.f16_sat(w) if kind == "fp16" else w.to(torch.bfloat16)


@pytest.mark.parametrize("kind", ["bf16", "fp16"])
def test_sgd_momentum_dyadic_three_steps(cuda, kind):
    """Three steps with accum carried, dyadic lr / mu / wd / gscale and gradients: w and accum equal the unrounded float64
    update after every step; the 16-bit copy equals the rounding of the master, with planted ties (RNE) and, in the first
    elements, NaN / +-inf gradients and masters beyond the fp16 range (saturation, NaN kept)."""
    H = R.SGD_DYADIC
    n = (1 << 20) + 5
    plan = R.ew_plan(n)
    print(f"n={n}: {plan['grid']} CTAs, {plan['items_per_thread']} items per thread, ragged {plan['ragged']}")
    assert plan["items_per_thread"] >= 4 and plan["ragged"]
    g = torch.Generator().manual_seed(11)
    S = 6                                                                       # special elements
    w = R.dyadic((n,), -1, 1, 2.0 ** -11, g)
    w[:S] = torch.tensor([0.5, 0.5, 0.5, 1e5, -1e5, 70000.0])
    acc = R.dyadic((n,), -1, 1, 2.0 ** -4, g)
    dw, dacc = w.to(cuda), acc.to(cuda)
    ties = 0
    for step in range(3):
        grad, tie = R.sgd_step_operands(w[S:], acc[S:], g, kind)
        special = [float("nan"), float("inf"), -float("inf")] if step == 0 else [0.0] * 3      # then NaN / inf propagate
        grad = torch.cat([torch.tensor(special + [0.0, 0.0, 0.0]), grad])
        ties += int(tie.sum())
        w64, a64 = R.sgd_f64(w, acc, grad, **H)
        w, acc = R.sgd_fp32(w, acc, grad, **H)
        assert torch.equal(w[S:].double(), w64[S:]) and torch.equal(acc[S:].double(), a64[S:])
        copy = _sgd(dw, dacc, grad.to(cuda), H, kind)
        assert_same(dw.cpu(), w, f"step {step}: w")
        assert_same(dacc.cpu(), acc, f"step {step}: accum")
        assert_same(copy.cpu().float(), _copy_ref(w, kind).float(), f"step {step}: {kind} copy")
        if step == 0:
            print(f"special masters {w[:S].tolist()} -> {kind} copies {copy[:S].tolist()}")
            assert torch.isnan(w[0]) and w[1].item() == -math.inf and w[2].item() == math.inf
            if kind == "fp16":
                assert torch.isnan(copy[0]) and bool(copy[1:S].float().abs().eq(65504).all())
    print(f"planted ties {ties}")
    assert ties > 1000


def test_sgd_momentum_realistic_fc6(cuda):
    """lr 0.001, mu 0.9, wd 1e-4 at fc6's 102,760,448 elements plus 3 (neither a multiple of 4 nor of the grid stride), from a
    non-zero accum (the momentum term): w, accum and the fp16 copy equal an exact fp32 emulation of the kernel's fmaf sequence
    on the CPU."""
    H = dict(lr=0.001, mu=0.9, wd=1e-4, gscale=1.0)
    n = 25088 * 4096 + 3
    plan = R.ew_plan(n)
    print(f"n={n}: {plan['grid']} CTAs, {plan['items_per_thread']} items per thread, ragged {plan['ragged']}")
    assert plan["ragged"] and n % 4 != 0
    g = torch.Generator(device=cuda).manual_seed(12)
    dw = torch.randn(n, generator=g, device=cuda) * 0.01
    dacc = torch.randn(n, generator=g, device=cuda) * 1e-3
    grad = torch.randn(n, generator=g, device=cuda) * 1e-3
    w, acc = R.sgd_fp32_chunked(dw.cpu(), dacc.cpu(), grad.cpu(), **H)
    copy = _sgd(dw, dacc, grad, H, "fp16")
    assert torch.equal(dw.cpu(), w), "w"
    assert torch.equal(dacc.cpu(), acc), "accum"
    assert torch.equal(copy.cpu(), R.f16_sat(w)), "fp16 copy"


def test_trainer_update_twice(cuda):
    """Trainer.update twice on synthetic gradients: every master and accum equals the emulated MomentumOptimizer step
    (fp32 fmaf, bit for bit), every tensor-core copy its rounding, and every derived copy (input-gradient weights, transposed
    fc weights, the conv1_1 tile) its re-derivation from the new masters."""
    from posecnn_b200 import conv
    from posecnn_b200.train import CONV_NAMES, SCORE_HEADS, Trainer
    from tests.train_ref import make_net
    net = make_net(cuda)
    lr, mu, wd = 0.01, 0.9, 1e-4
    tr = Trainer(net, lr=lr, momentum=mu, weight_decay=wd)
    g = torch.Generator(device=cuda).manual_seed(13)
    H = dict(lr=lr, mu=mu, wd=wd, gscale=1.0)
    print(f"{len(tr.master)} parameters, {sum(v.numel() for v in tr.master.values())} elements")
    for step in range(2):
        grads = {k: torch.randn(v.shape, generator=g, device=cuda) * 1e-3 for k, v in tr.master.items()}
        want = {k: R.sgd_fp32(tr.master[k], tr.accum[k], grads[k], **H) for k in tr.master}
        tr.update(grads)
        torch.cuda.synchronize()
        for k, (w, a) in want.items():
            assert torch.equal(tr.master[k], w), f"step {step}: {k} master"
            assert torch.equal(tr.accum[k], a), f"step {step}: {k} accum"
            if tr.tc[k] is not None:
                assert torch.equal(tr.tc[k], R.f16_sat(w) if tr.tc[k].dtype == torch.float16 else w.to(torch.bfloat16)), k
        del want
        M = tr.master
        for name in CONV_NAMES[1:]:
            assert torch.equal(tr.dg[name], conv.hwio_to_tc_dgrad(tr.to_tf(name + "/w", M[name + "/w"]))), name
        for name in SCORE_HEADS + ("score", "vertex_pred"):
            assert torch.equal(tr.dg[name], M[name + "/w"].to(torch.bfloat16).t().contiguous()), name
        for name in tr.fc_names:
            assert torch.equal(tr.fc_t[name], R.f16_sat(M[name + "/w"]).t().contiguous()), name
        assert torch.equal(tr.conv1_tc, conv.conv1_1_weights_to_tc(tr.to_tf("conv1_1/w", M["conv1_1/w"])))
