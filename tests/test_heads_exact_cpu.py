"""CPU rehearsal of tests/heads_ref.py: each float64 reference of the FCN-head kernels equals an fp32 torch computation of the
same operation in a different order (dense conv2d / conv_transpose2d with the bilinear filter), bit for bit, on dyadic
operands; the bit budget refuses an operand range that is too wide; the launch plans reproduce the formulas of
csrc/heads.cu and csrc/train_bwd.cu (and the workspace the library itself asks for)."""
import ctypes
import re

import pytest
import torch
import torch.nn.functional as F

from tests import heads_ref as R


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def bilinear_filter(C, k):
    k1 = torch.tensor(R.bilinear_taps(k))
    return (k1[:, None] * k1[None, :])[None, None].expand(C, 1, k, k).contiguous()


def up2_fp32(a5):
    C = a5.shape[3]
    return nhwc(F.conv_transpose2d(nchw(a5), bilinear_filter(C, 4), stride=2, padding=1, groups=C))


def test_taps_are_the_kernel_filters():
    assert R.bilinear_taps(4) == [0.25, 0.75, 0.75, 0.25]
    assert R.bilinear_taps(16) == [(2 * i + 1) / 16 for i in range(8)] + [(15 - 2 * i) / 16 for i in range(8)]
    assert torch.equal(R.up_matrix(3, 2).sum(0), torch.tensor([1.75, 2.0, 1.75], dtype=torch.float64))   # border columns see 3 taps


def test_add_up2_and_adjoint_references():
    g = torch.Generator().manual_seed(0)
    for h, w in ((6, 10), (10, 14)):                                       # even and odd conv5 grids
        a4 = R.dyadic((2, h, w, 16), -3, 3, 1, g)
        a5 = R.dyadic((2, h // 2, w // 2, 16), -3, 3, 1, g)
        ref, budget = R.add_up2(a4, a5, 1.0)
        assert 0 < budget < 2 ** 10
        assert torch.equal(ref, (a4 + up2_fp32(a5)).double())
        dadd = R.dyadic((2, h, w, 16), -3, 3, 1, g)
        y5 = R.dyadic((2, h // 2, w // 2, 16), -1, 1, 1, g)
        want = nhwc(F.conv2d(nchw(dadd), bilinear_filter(16, 4), stride=2, padding=1, groups=16))
        d5, _ = R.up2_bwd(dadd, y5, 1.0)
        assert torch.equal(d5, (want * (y5 > 0)).double())
        assert torch.equal(R.up2_bwd(dadd, None, 1.0)[0], want.double())


def test_pack_and_lowres_heads_references():
    g = torch.Generator().manual_seed(1)
    B, h, w, Cs, Cv = 2, 6, 8, 64, 128
    for C in (2, 6, 22):
        s4, s5 = R.dyadic((B, h, w, Cs), -3, 3, 1, g), R.dyadic((B, h // 2, w // 2, Cs), -3, 3, 1, g)
        v4, v5 = R.dyadic((B, h, w, Cv), -3, 3, 1, g), R.dyadic((B, h // 2, w // 2, Cv), -3, 3, 1, g)
        Ws, Wv = R.dyadic((Cs, C), -2, 2, 0.125, g), R.dyadic((Cv, 3 * C), -2, 2, 0.125, g)
        add_s, add_v = s4 + up2_fp32(s5), v4 + up2_fp32(v5)
        ref, budget = R.lowres_heads(s4, s5, v4, v5, Ws, Wv, C, 1.0, 0.125)
        assert 0 < budget < R.LIMIT
        assert torch.equal(ref, torch.cat([torch.einsum("nhwk,kc->nhwc", add_s, Ws), torch.einsum("nhwk,kc->nhwc", add_v, Wv)], 3).double())
        folded, _ = R.lowres_heads(s4, s5, v4, v5, Ws, None, C, 1.0, 0.125)
        assert torch.equal(folded[..., C:], add_v[..., :3 * C].double()) and torch.equal(folded[..., :C], ref[..., :C])
        packed = R.pack_lowres(s4, v4, C)
        assert packed.shape == (B, h, w, 4 * C) and torch.equal(packed, torch.cat([s4[..., :C], v4[..., :3 * C]], 3).double())


def test_up8_heads_reference():
    g = torch.Generator().manual_seed(2)
    B, h, w = 2, 5, 7
    for C in (2, 6):
        lowres = R.dyadic((B, h, w, 4 * C), -1, 1, 0.125, g)
        bs, bv = R.dyadic((C,), -0.5, 0.5, 0.125, g), R.dyadic((3 * C,), -1, 1, 0.125, g)
        ref = R.up8_heads(lowres, bs, bv, C, 0.125)
        up = nhwc(F.conv_transpose2d(nchw(lowres), bilinear_filter(4 * C, 16), stride=8, padding=4, groups=4 * C))
        assert torch.equal(ref["score"], torch.relu(up[..., :C] + bs).double())
        assert torch.equal(ref["vertex"], (up[..., C:] + bv).double())
        assert torch.equal(ref["label"], torch.argmax(ref["score"], -1))          # torch.argmax: the first maximal index
        zero = (ref["score"] == 0).all(-1)
        assert bool(zero.any()) and bool((ref["label"][zero] == 0).all())          # ReLU zeros: all-class ties
        bound = R.softmax_bound(ref["prob"], C)
        assert bool((bound < 1e-6).all()) and bool((bound > 0).all())


@pytest.mark.parametrize("coord", [False, True])
def test_up8_bwd_reference(coord):
    """The adjoint reference against the formulas of lib/fcn/train.py written in fp32 torch and a dense stride-8 conv2d."""
    g = torch.Generator().manual_seed(3 + coord)
    B, h, w, C = 2, 5, 7, 6
    P = R.up8_bwd_problem(B, h, w, C, coord, g)
    H, W = 8 * h, 8 * w
    for sigma, thr in ((1.0, 1.0), (2.0, 0.5)):
        ref = R.up8_bwd(P, sigma, thr, 2.0 ** -10)
        assert 0 < ref["budget"] < R.LIMIT
        gt = P["gt"].long()
        valid = (gt >= 0) & (gt < C)
        g0 = torch.where(valid, gt, 0)
        sel = valid & ((gt > 0) | (P["prob"][..., 0] < thr))
        d_s = (1.0 / 1024) * sel[..., None] * (P["prob"] - F.one_hot(g0, C).float()) * (P["score"] > 0)
        listed = valid & (gt > 0) & (P["centers"][torch.arange(B)[:, None, None], g0, 2] > 0)
        pv = P["pv"].float().view(B, H, W, C, 3).gather(3, g0[..., None, None].expand(B, H, W, 1, 3))[..., 0, :]
        if coord:
            ext = P["extents"][g0]
            a = torch.where(ext > 0, 1.0 / ext.clamp(min=1e-30), torch.zeros(()))
            tg = a * P["vertmap"] + torch.where(ext > 0, 0.5, 0.0)
        else:
            cen = P["centers"][torch.arange(B)[:, None, None], g0]
            ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
            dx, dy = cen[..., 0].double() - xs, cen[..., 1].double() - ys
            nrm = (dx * dx + dy * dy).sqrt() + 1e-10
            tg = torch.stack([(dx / nrm).float(), (dy / nrm).float(), torch.zeros(B, H, W)], -1)
        diff = 4.0 * (pv - tg)
        dt = torch.where(diff.abs() < 1.0 / sigma ** 2, diff * sigma ** 2, diff.sign())
        d_own = (2.0 / 1024) * 4.0 * dt * listed[..., None]
        d_v = torch.zeros(B, H, W, C, 3).scatter_(3, g0[..., None, None].expand(B, H, W, 1, 3), d_own[..., None, :]).view(B, H, W, 3 * C)
        d_up = torch.cat([d_s, d_v], 3)
        want = nhwc(F.conv2d(nchw(d_up), bilinear_filter(4 * C, 16), stride=8, padding=4, groups=4 * C))
        assert torch.equal(ref["d_sc"], want[..., :C].double()) and torch.equal(ref["d_vt"], want[..., C:].double())
        assert torch.equal(ref["dbias"], d_up.sum((0, 1, 2)).double())
        assert bool(ref["d_vt"].ne(0).any()) and bool(ref["d_sc"].ne(0).any())


def test_loss_reference():
    g = torch.Generator().manual_seed(4)
    B, H, W, C = 2, 16, 24, 6
    s = R.dyadic((B, H, W, C), -4, 4, 0.125, g)
    s[0, 0, :4] = torch.tensor([80.0, -80.0, 0.0, 0.0, 0.0, 0.0])
    prob = R.dyadic((B, H, W, C), 0, 1, 0.125, g)
    gt = R.int_operands((B, H, W), -1, C - 1, g).to(torch.int32)
    loss, n, bound, logsm = R.loss_cls_hard_raw(s, prob, gt, 0.5)
    sel = (gt >= 0) & ((gt > 0) | (prob[..., 0] < 0.5))
    want = -torch.log_softmax(s.double(), -1).gather(-1, gt.clamp(min=0).long()[..., None])[..., 0][sel].sum() / int(sel.sum())
    assert n == int(sel.sum()) and abs(loss - float(want)) <= 1e-12 * abs(float(want))
    assert 0 < bound < 1e-5
    assert R.loss_cls_hard_raw(s, prob, torch.full_like(gt, -1), 0.5)[:2] == (0.0, 0)


def test_bit_budget_refuses_a_wide_operand_range():
    g = torch.Generator().manual_seed(5)
    a4 = R.dyadic((1, 4, 4, 8), -3, 3, 1, g)
    wide = R.dyadic((1, 2, 2, 8), -2 ** 21, 2 ** 21, 1, g)
    with pytest.raises(R.BudgetExceeded, match="add_up2"):
        R.add_up2(a4, wide, 1.0)
    with pytest.raises(R.BudgetExceeded, match="up8_heads"):
        R.up8_heads(R.dyadic((1, 2, 3, 8), -2 ** 14, 2 ** 14, 0.125, g), torch.zeros(2), torch.zeros(6), 2, 0.125)
    with pytest.raises(AssertionError, match="grid"):
        R.add_up2(a4, a4[:, :2, :2] + 0.5, 1.0)
    P = R.up8_bwd_problem(1, 4, 6, 2, False, g, count=1.0)        # normaliser 1: d up on a grid 2^10 times finer than the range
    with pytest.raises(R.BudgetExceeded, match="up8_bwd"):
        R.up8_bwd(P, 1.0, 0.5, 2.0 ** -10, prob_unit=2.0 ** -20)


def test_coverage_helpers(native_lib):
    p = R.up8_bwd_plan(2, 60, 80, 22)
    assert (p["strips"], p["bands"], p["last_strip_cells"], p["last_band_rows"], p["threads"]) == (20, 4, 4, 12, 440)
    p = R.up8_bwd_plan(2, 60, 80, 50)
    assert (p["kernel"], p["threads"], p["smem"]) == ("<0>", 1000, 88200)                    # the largest class count: ~88 KB
    p = R.up8_bwd_plan(2, 60, 80, 2)
    assert (p["kernel"], p["strip"], p["strips"], p["threads"]) == ("<2>", 16, 5, 136)
    p, p2 = R.up8_bwd_plan(2, 37, 27, 12), R.up8_bwd_plan(2, 37, 27, 2)
    assert (p["strips"], p["last_strip_cells"], p["bands"], p["last_band_rows"]) == (7, 3, 3, 5)
    assert (p2["strips"], p2["last_strip_cells"]) == (2, 11)
    # the workspace the entry point asks for (its "workspace too small (have < need)" check runs before any launch)
    buf = ctypes.create_string_buffer(64)
    for B, h, w, C in ((2, 60, 80, 50), (2, 37, 27, 2), (2, 37, 27, 12)):
        rc = native_lib.pcnn_up8_heads_bwd(buf, buf, buf, buf, 1.0, 1.0, buf, buf, buf, None, None, buf, 1.0, 1.0, 1.0, B, h, w, C, 64,
                                           R.vertex_stride(C), buf, buf, buf, buf, 16, None)
        assert rc == -1
        need = re.search(rb"workspace too small \(16 < (\d+)\)", native_lib.pcnn_last_error())
        assert need and int(need.group(1)) == R.up8_bwd_plan(B, h, w, C)["workspace"], native_lib.pcnn_last_error()
    B, p = R.ew_batch_for_coverage(60 * 80 * 64 // 8)                  # add_up2, 64 channels
    assert (B, p["blocks"], p["iters"]) == (8, 1056, 2)
    B, p = R.ew_batch_for_coverage(30 * 40 * 64 // 8)                  # up2_bwd, 64 channels: one thread per conv5 pixel and 8 channels
    assert (B, p["iters"]) == (29, 2)
    p = R.lowres_heads_plan(4, 60, 80, 50)
    assert (p["blocks"], p["groups"], p["groups_per_warp"], p["full_passes"], p["tail_passes"]) == (264, 2400, 2, 4, 3)
    p = R.lowres_heads_plan(15, 60, 80, 22, folded=True)
    assert (p["blocks"], p["groups_per_warp"], p["full_passes"]) == (1056, 2, 0)
    assert R.lowres_heads_plan(5, 62, 82, 6)["ragged_group"]
    assert R.up8_heads_plan(2, 60, 80, 58, label_only=True)["kernel"] == "k_up8_label"
    assert R.up8_heads_plan(2, 60, 80, 64, label_only=True)["kernel"] == "k_up8_heads"     # 11 w C floats > 200 KB
    assert R.up8_heads_plan(2, 60, 80, 22)["segments"] == 4


@pytest.mark.parametrize("C", [2, 6, 9, 22, 50])
def test_up8_bwd_workspace_query(native_lib, C):
    """pcnn_up8_heads_bwd_workspace_bytes is the size heads_ref.up8_bwd_plan restates (4C floats per CTA of its strips and 16-row
    bands) at 480 x 640, at 296 x 216 (partial last strip and band) and on an odd batch, and the size the entry point checks."""
    nbytes = ctypes.c_size_t(0)
    buf = ctypes.create_string_buffer(64)
    for B, h, w in ((2, 60, 80), (2, 37, 27), (5, 37, 27)):
        assert native_lib.pcnn_up8_heads_bwd_workspace_bytes(B, h, w, C, ctypes.byref(nbytes)) == 0
        assert nbytes.value == R.up8_bwd_plan(B, h, w, C)["workspace"], (B, h, w)
        rc = native_lib.pcnn_up8_heads_bwd(buf, buf, buf, buf, 1.0, 1.0, buf, buf, buf, None, None, buf, 1.0, 1.0, 1.0, B, h, w, C, 64,
                                           R.vertex_stride(C), buf, buf, buf, buf, nbytes.value - 1, None)
        assert rc == -1 and f"workspace too small ({nbytes.value - 1} < {nbytes.value})".encode() in native_lib.pcnn_last_error()
    assert native_lib.pcnn_up8_heads_bwd_workspace_bytes(2, 60, 80, C, None) == -1
    assert native_lib.pcnn_up8_heads_bwd_workspace_bytes(0, 60, 80, C, ctypes.byref(nbytes)) == -1
