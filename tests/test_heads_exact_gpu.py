"""The FCN-head kernels of the training step and of inference, bit for bit against float64 references at training shapes.

Operands lie on dyadic grids (tests/heads_ref.py) so that every fp32 sum in the kernels is exact in any order; each
reference checks that condition (its bit budget) and the kernel's output must equal the reference rounded once: bf16
round-to-nearest-even for d_sc / d_vt / add / d5, fp32 for everything else.  The exceptions are the softmax probabilities
and the classification loss, which go through expf / logf and are held to bounds derived from those functions' documented
errors.  Kernel-vs-reference comparisons are by value (+0 == -0); kernel-vs-kernel comparisons (two launches) are by bit
pattern.  Each test prints the launch plan it covered and asserts that coverage.
The rel-L2 tests of the same kernels (test_backward_gpu.py, test_network_gpu.py, ...) stay: they cover random-float
rounding, a different question."""
import pytest
import torch

from tests import heads_ref as R

pytestmark = pytest.mark.gpu


def bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_same(got, want, what):
    bad = got != want
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} values differ; first at {bad.nonzero()[0].tolist()}: "
                                 f"{got[tuple(bad.nonzero()[0])].item()} != {want[tuple(bad.nonzero()[0])].item()}")


def bf16(ref):
    return ref.float().to(torch.bfloat16)        # exact in fp32 (checked budget), then one round-to-nearest-even


# ---------------------------------------------------------------------------------------------------------------------
# 1. the up-sampling adjoint of both losses (k_up8_bwd_strip + k_sum_partials)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("coord", [False, True], ids=["2d", "3d"])
@pytest.mark.parametrize("h,w", [(60, 80), (37, 27)])
@pytest.mark.parametrize("C", [2, 6, 12, 22, 50])
def test_up8_bwd_exact(cuda, C, h, w, coord):
    """pcnn_up8_heads_bwd in both target modes at 480 x 640 (ragged last band of 12 rows) and 296 x 216 (partial last strip of the 4-
    and the 16-cell kernels, last band of 5 rows), B = 2, sigma 1 / threshold 1 and sigma 2 / threshold 1/2: d_sc, d_vt
    and d bias exact; padding channels 0; two launches bit-identical."""
    B, Cv = 2, R.vertex_stride(C)
    plan = R.up8_bwd_plan(B, h, w, C)
    print(f"C={C} {h}x{w} {'3d' if coord else '2d'}: kernel {plan['kernel']} strip {plan['strip']}: {plan['strips']} strips x "
          f"{plan['bands']} bands x {B} images = {plan['ctas']} CTAs of {plan['threads']} threads; last strip {plan['last_strip_cells']} "
          f"cells, last band {plan['last_band_rows']} rows")
    assert plan["last_band_rows"] < 16 and plan["strips"] >= 2 and plan["bands"] >= 3
    if (h, w) == (37, 27):
        assert plan["last_strip_cells"] < plan["strip"]
    g = torch.Generator().manual_seed(1000 * C + h + 2 * coord)
    P = R.up8_bwd_problem(B, h, w, C, coord, g, device=cuda)
    gt, p0 = P["gt"], P["prob"][..., 0]
    assert bool((gt == -1).any() and (gt >= C).any() and (gt < -1).any() and (P["score"] == 0).any())
    for sigma, thr in ((1.0, 1.0), (2.0, 0.5)):
        bg = gt == 0
        assert bool((bg & (p0 < thr)).any() and (bg & (p0 == thr)).any() and (bg & (p0 == thr - 0.125)).any())
        ref = R.up8_bwd(P, sigma, thr, 2.0 ** -10)
        print(f"  sigma={sigma} threshold={thr}: bit budget {ref['budget']:.0f} of 2^24")
        e_sc, e_vt, ebias = R.run_up8_bwd(P, sigma, thr, Cv)
        again = R.run_up8_bwd(P, sigma, thr, Cv)
        torch.cuda.synchronize()
        for a, b in zip((e_sc, e_vt, ebias), again):
            assert torch.equal(bits(a), bits(b)), "two launches differ"
        assert_same(e_sc[..., :C], bf16(ref["d_sc"]), "d_sc")
        assert_same(e_vt[..., :3 * C], bf16(ref["d_vt"]), "d_vt")
        assert_same(ebias, ref["dbias"].float(), "dbias")
        assert not bool(e_sc[..., C:].float().ne(0).any()) and not bool(e_vt[..., 3 * C:].float().ne(0).any()), "padding channels"
        assert bool(ref["d_vt"].ne(0).any()) and bool(ref["dbias"][C:].ne(0).any())


# ---------------------------------------------------------------------------------------------------------------------
# 2. add = a4 + up2(a5) and its adjoint with the ReLU mask; 3. the 1/8-resolution pack
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(60, 80), (62, 82)])
@pytest.mark.parametrize("C", [64, 128])
def test_add_up2_and_adjoint_exact(cuda, C, h, w):
    """pcnn_add_up2_bf16 / pcnn_up2_bwd_bf16 at conv4 60 x 80 (conv5 30 x 40) and 62 x 82 (odd conv5 grid 31 x 41) on small
    integers, batches chosen so that the grid-stride loop runs at least twice; masks with exact zeros (the test is y5 > 0)."""
    from posecnn_b200 import heads
    g = torch.Generator().manual_seed(C + h)
    Bf, pf = R.ew_batch_for_coverage(h * w * C // 8)
    Bb, pb = R.ew_batch_for_coverage((h // 2) * (w // 2) * C // 8)
    print(f"C={C} {h}x{w}: add_up2 B={Bf}: {pf['total']} items on {pf['blocks']} blocks, {pf['iters']} grid-stride iterations; "
          f"up2_bwd B={Bb}: {pb['total']} items, {pb['iters']} iterations")
    assert pf["iters"] >= 2 and pb["iters"] >= 2
    # operands stay referenced while the kernels run: a temporary's block could be handed to the next allocation
    a4 = R.dyadic((Bf, h, w, C), -3, 3, 1, g).to(cuda).bfloat16()
    a5 = R.dyadic((Bf, h // 2, w // 2, C), -3, 3, 1, g).to(cuda).bfloat16()
    out = heads.add_up2(a4, a5)
    ref, budget = R.add_up2(a4, a5, 1.0)
    assert_same(out, bf16(ref), "add_up2")
    dadd = R.dyadic((Bb, h, w, C), -3, 3, 1, g).to(cuda).bfloat16()
    y5 = R.dyadic((Bb, h // 2, w // 2, C), -1, 1, 1, g).to(cuda).bfloat16()
    assert bool((y5 == 0).any())
    for mask in (y5, None):
        d5 = heads.up2_bwd(dadd, mask)
        ref5, b5 = R.up2_bwd(dadd, mask, 1.0)
        assert_same(d5, bf16(ref5), "up2_bwd" + (" (masked)" if mask is not None else ""))
    print(f"  bit budgets {budget:.0f}, {b5:.0f} of 2^24")


@pytest.mark.parametrize("C", [2, 22, 50])
def test_pack_lowres_exact(cuda, C):
    """pcnn_pack_lowres: an exact copy of the first C score channels (stride 64) and 3C vertex channels (stride Cv)."""
    from posecnn_b200 import heads
    h, w, Cs, Cv = 60, 80, 64, R.vertex_stride(C)
    B, plan = R.ew_batch_for_coverage(h * w * 4 * C)
    print(f"C={C} Cv={Cv}: B={B}, {plan['total']} floats on {plan['blocks']} blocks, {plan['iters']} grid-stride iterations")
    assert plan["iters"] >= 2
    g = torch.Generator().manual_seed(C)
    sc = torch.randn(B, h, w, Cs, generator=g).to(torch.bfloat16).to(cuda)
    vt = torch.randn(B, h, w, Cv, generator=g).to(torch.bfloat16).to(cuda)
    out = heads.pack_lowres(sc, vt, C)
    assert torch.equal(bits(out), bits(R.pack_lowres(sc, vt, C).float()))


# ---------------------------------------------------------------------------------------------------------------------
# 4. the 1x1 heads at 1/8 resolution (k_lowres_heads)
# ---------------------------------------------------------------------------------------------------------------------
_LR = [(C, False) for C in (2, 6, 22, 50)] + [(C, True) for C in (2, 6, 22, 42)]


@pytest.mark.parametrize("h,w", [(60, 80), (62, 82)])
@pytest.mark.parametrize("C,folded", _LR, ids=[f"{C}-{'folded' if f else 'unfolded'}" for C, f in _LR])
def test_lowres_heads_exact(cuda, C, folded, h, w):
    """pcnn_lowres_heads at 60 x 80 and 62 x 82 (B h w not a multiple of 8), batches chosen so that warps take at least two
    8-pixel groups (block caps kNumSMs x 2 unfolded, x 8 folded).  Unfolded C = 50 runs four full vertex passes and three
    tail passes.  Folded mode needs 3C <= Cv = 128, so its largest class count is 42."""
    from posecnn_b200 import heads
    Cs, Cv = 64, 128
    B = 15 if folded else (4 if (h, w) == (60, 80) else 5)
    plan = R.lowres_heads_plan(B, h, w, C, Cs, Cv, folded)
    print(f"C={C} {'folded' if folded else 'unfolded'} {h}x{w} B={B}: {plan['groups']} groups on {plan['warps']} warps, up to "
          f"{plan['groups_per_warp']} per warp; {plan['full_passes']} full + {plan['tail_passes']} tail passes, ragged last group "
          f"{plan['ragged_group']}")
    assert plan["groups_per_warp"] >= 2
    assert plan["ragged_group"] == ((h, w) == (62, 82))
    g = torch.Generator().manual_seed(10 * C + h + folded)
    s4, s5 = R.dyadic((B, h, w, Cs), -3, 3, 1, g), R.dyadic((B, h // 2, w // 2, Cs), -3, 3, 1, g)
    v4, v5 = R.dyadic((B, h, w, Cv), -3, 3, 1, g), R.dyadic((B, h // 2, w // 2, Cv), -3, 3, 1, g)
    Ws = R.dyadic((Cs, C), -2, 2, 0.125, g).to(cuda)
    Wv = None if folded else R.dyadic((Cv, 3 * C), -2, 2, 0.125, g).to(cuda)
    s4, s5, v4, v5 = (t.to(cuda).bfloat16() for t in (s4, s5, v4, v5))
    out = heads.lowres_heads(s4, s5, v4, v5, Ws, Wv, C)
    ref, budget = R.lowres_heads(s4, s5, v4, v5, Ws, Wv, C, 1.0, 0.125)
    print(f"  bit budget {budget:.0f} of 2^24")
    assert_same(out, ref.float(), "lowres_heads")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the dense heads (k_up8_heads, k_up8_label)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [2, 6, 22, 50, 64])
def test_up8_heads_exact(cuda, C):
    """pcnn_up8_heads at 480 x 640, B = 2: vertex and score exact, label the first-index arg-max (exact ties from coarse
    scores and all-class ties from ReLU zeros), prob within the softmax bound; the label-only call (k_up8_label, or at
    C = 64, where 11 w C floats exceed its shared memory, k_up8_heads without outputs) gives the same labels."""
    from posecnn_b200 import heads
    B, h, w = 2, 60, 80
    H, W = 8 * h, 8 * w
    full, lab = R.up8_heads_plan(B, h, w, C), R.up8_heads_plan(B, h, w, C, label_only=True)
    print(f"C={C}: {full['kernel']} grid {full['grid']} ({full['segments']} segments, ragged {full['ragged_segment']}); label-only: "
          f"{lab['kernel']} grid {lab['grid']}, {lab['smem']} B of shared memory")
    assert lab["kernel"] == ("k_up8_heads" if C > 58 else "k_up8_label")
    g = torch.Generator().manual_seed(200 + C)
    lowres = R.dyadic((B, h, w, 4 * C), -1, 1, 0.125, g)
    lowres[..., :C] = R.dyadic((B, h, w, C), -1, 1, 0.5, g)                # coarse scores: exact ties between classes
    for y0, x0 in ((8, 8), (40, 60), (h - 3, w - 3)):
        lowres[:, y0:y0 + 3, x0:x0 + 3, :C] = -1.0                          # every class negative: ReLU zeros tie across classes
    bs =R.dyadic((C,), -0.25, 0.25, 0.125, g) * (torch.arange(C) % 2)    # half the classes without bias
    bv = R.dyadic((3 * C,), -1, 1, 0.125, g)
    lowres, bs, bv = lowres.to(cuda), bs.to(cuda), bv.to(cuda)
    label = torch.full((B, H, W), -7, dtype=torch.int32, device=cuda)
    _, vertex, prob, score = heads.up8_heads(lowres, bs, bv, out=(label, torch.empty((B, H, W, 3 * C), device=cuda),
                                                                  torch.empty((B, H, W, C), device=cuda), torch.empty((B, H, W, C), device=cuda)))
    label2 = heads.up8_heads(lowres, bs, bv, out=(torch.full((B, H, W), -7, dtype=torch.int32, device=cuda), None, None, None))[0]
    ref = R.up8_heads(lowres, bs, bv, C, 0.125)
    print(f"  bit budget {ref['budget']:.0f} of 2^24")
    assert_same(vertex, ref["vertex"].float(), "vertex")
    assert_same(score, ref["score"].float(), "score")
    del vertex
    top2 = ref["score"].topk(2, -1).values
    ties, zeros = (top2[..., 0] == top2[..., 1]) & (top2[..., 0] > 0), (top2[..., 0] == 0)
    print(f"  {int(ties.sum())} pixels with tied positive maxima, {int(zeros.sum())} all-zero pixels")
    assert bool(ties.any()) and bool(zeros.any())
    assert_same(label, ref["label"].int(), "label")
    assert_same(label2, ref["label"].int(), "label (label-only call)")
    err = (prob.double() - ref["prob"]).abs()
    bound = R.softmax_bound(ref["prob"], C)
    print(f"  prob: max |err| / bound = {float((err / bound).max()):.3f}")
    assert bool((err <= bound).all()), f"prob outside the softmax bound at {int((err > bound).sum())} values"


# ---------------------------------------------------------------------------------------------------------------------
# 6. the classification loss of the training step (k_loss_cls_hard_raw)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,thr", [pytest.param(C, 0.5, id=str(C)) for C in (2, 22, 50)] +
                         [pytest.param(C, t, id=f"{C}-thr{t}") for t in (1.0, 0.4) for C in (2, 22, 50)])
def test_loss_cls_hard_raw(cuda, C, thr):
    """train_ops.loss_cls (pcnn_loss_cls_hard_raw_fwd, the step's loss_cls) at 2 x 480 x 640: count exact, loss within the bound
    derived from fp32 expf / logf (heads_ref.loss_cls_hard_raw) of the float64 log-softmax reference, also with raw scores of +-80
    where an unshifted exp overflows; two launches bit-identical; an all-ignore batch gives 0 and 0; and the un-fused composition
    through the Hardlabel op (its mask times the float64 log-softmax) selects the same pixels and agrees within 1e-5 relative."""
    from posecnn_b200.hard_label_layer import hard_label_op
    from posecnn_b200.train_ops import loss_cls
    B, H, W = 2, 480, 640
    npix = B * H * W
    blocks = R.NUM_SMS * 4
    print(f"C={C}, threshold {thr}: {npix} pixels on {blocks} x 256 threads, {-(-npix // (blocks * 256))} grid-stride iterations")
    g = torch.Generator().manual_seed(300 + C)
    score = R.dyadic((B, H, W, C), -8, 8, 0.125, g)
    hot = R.int_operands((B, H, W), 0, 19, g) == 0                          # 5 % of the pixels: one channel +80, one -80
    c_hi = R.int_operands((B, H, W), 0, C - 1, g).long()
    c_lo = (c_hi + 1) % C
    score[hot] = score[hot].scatter(-1, c_hi[hot][:, None], 80.0).scatter(-1, c_lo[hot][:, None], -80.0)
    prob = R.dyadic((B, H, W, C), 0, 1, 0.125, g)
    gt = R.int_operands((B, H, W), -2, C, g).to(torch.int32)                # -2 and C: out of range, ignored like -1
    score, prob, gt, hot = score.to(cuda), prob.to(cuda), gt.to(cuda), hot.to(cuda)
    a = loss_cls(score, prob, gt, thr)
    b = loss_cls(score, prob, gt, thr)
    loss, n, bound, logsm = R.loss_cls_hard_raw(score, prob, gt, thr)
    sel = ((gt >= 0) & (gt < C) & ((gt > 0) | (prob[..., 0] < thr)))
    assert bool((sel & hot & (score.gather(-1, gt.clamp(0, C - 1).long()[..., None])[..., 0] == -80)).any())
    print(f"  loss {a[0].item():.9f} ref {loss:.9f} |err| {abs(a[0].item() - loss):.3e} bound {bound:.3e}; count {int(a[1].item())}")
    assert torch.equal(bits(a), bits(b)), "two launches differ"
    assert a[1].item() == n
    assert abs(a[0].item() - loss) <= bound
    m = hard_label_op.hard_label(prob, gt, thr).double()
    comp = float(-(m * logsm).sum() / (m.sum() + 1e-10))
    assert m.sum().item() == n
    assert abs(a[0].item() - comp) <= 1e-5 * abs(comp)
    none = loss_cls(score, prob, torch.full_like(gt, -1), thr)
    assert none.tolist() == [0.0, 0.0]
