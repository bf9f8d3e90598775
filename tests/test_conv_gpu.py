"""wgmma implicit-GEMM convolution vs a plain PyTorch fp32 reference of the same op
(tf.nn.conv2d semantics of lib/networks/network.py:159-188: NHWC x HWIO, SAME, stride 1, bias, ReLU).
Inputs and weights are rounded to bf16 first, so only the fp32 accumulation order and the final
bf16 rounding of the output differ: tolerance = 2 bf16 ulps of the output magnitude."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def ref_conv(x_bf16, w_hwio_bf16, bias, relu):
    x = x_bf16.float().permute(0, 3, 1, 2)
    w = w_hwio_bf16.float().permute(3, 2, 0, 1)
    y = F.conv2d(x, w, bias, padding=w.shape[2] // 2)
    if relu:
        y = F.relu(y)
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,bn", [
    (1, 8, 16, 64, 64, 3, 64),       # exactly one tile
    (2, 24, 48, 64, 64, 3, 64),      # conv1_2-like
    (1, 30, 40, 128, 128, 3, 128),   # ragged tiles (30 = 3*8+6, 40 = 2*16+8): zero-fill + clipped stores
    (2, 16, 32, 256, 256, 3, 256),
    (1, 15, 20, 512, 512, 3, 256),   # two N tiles
    (1, 16, 32, 128, 256, 3, 128),
    (2, 16, 16, 512, 128, 1, 128),   # 1x1 head
    (3, 37, 53, 64, 128, 3, 0),      # odd sizes, automatic N tile
])
def test_conv_tc_matches_fp32_reference(cuda, B, H, W, Cin, Cout, k, bn):
    from posecnn_b200 import conv
    g = torch.Generator(device="cpu").manual_seed(1234 + H + Cin)
    x = torch.randn((B, H, W, Cin), generator=g).to(torch.bfloat16).to(cuda)
    w = (torch.randn((k, k, Cin, Cout), generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16).to(cuda)
    bias = torch.randn((Cout,), generator=g).to(cuda)
    for relu in (True, False):
        y = conv.conv_bf16(x, conv.hwio_to_tc(w.float()), bias, k, relu, bn)
        torch.cuda.synchronize()
        want = ref_conv(x, w, bias, relu)
        err = (y.float() - want).abs()
        tol = 2 ** -7 * want.abs().clamp(min=1.0)          # 2 bf16 ulps
        assert (err <= tol).all(), f"max err {err.max().item():.4g} at |want| up to {want.abs().max().item():.3g}"
        rel_l2 = (err.pow(2).sum() / want.pow(2).sum()).sqrt().item()
        assert rel_l2 < 4e-3, rel_l2


def test_conv_small_cin_and_maxpool(cuda):
    from posecnn_b200 import conv
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randn((2, 20, 28, 3), generator=g).to(cuda)
    w = (torch.randn((3, 3, 3, 64), generator=g) * 0.3).to(cuda)
    b = torch.randn((64,), generator=g).to(cuda)
    y = conv.conv3x3_small_cin(x, w, b, True)
    want = F.relu(F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, padding=1)).permute(0, 2, 3, 1)
    assert ((y.float() - want).abs() <= 2 ** -7 * want.abs().clamp(min=1.0)).all()
    p = conv.maxpool2x2(y)
    wantp = F.max_pool2d(y.float().permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    assert torch.equal(p.float(), wantp)


@pytest.mark.parametrize("B,H,W,Cin,Cout,bn", [(2, 24, 48, 64, 64, 64), (1, 30, 44, 128, 128, 128), (1, 16, 32, 256, 256, 256),
                                             (2, 60, 80, 64, 128, 0)])
def test_conv_pool_fused(cuda, B, H, W, Cin, Cout, bn):
    """conv + bias + ReLU + 2x2/2 max pool fused in the epilogue == un-fused conv followed by the pool kernel (bit exact)."""
    from posecnn_b200 import conv
    g = torch.Generator(device="cpu").manual_seed(99 + H)
    x = torch.randn((B, H, W, Cin), generator=g).to(torch.bfloat16).to(cuda)
    w = conv.hwio_to_tc((torch.randn((3, 3, Cin, Cout), generator=g) * (2.0 / (9 * Cin)) ** 0.5).to(cuda))
    bias = torch.randn((Cout,), generator=g).to(cuda)
    want = conv.maxpool2x2(conv.conv_bf16(x, w, bias, 3, True, bn))
    got = conv.conv_pool_bf16(x, w, bias, 3, True, bn)
    torch.cuda.synchronize()
    assert got.shape == want.shape
    assert torch.equal(got, want)


@pytest.mark.parametrize("dtype,H,W", [(torch.uint8, 37, 53), (torch.float32, 37, 53), (torch.uint8, 37, 52), (torch.uint8, 48, 80),
                                       (torch.uint8, 8, 16)])
def test_conv1_fused_matches_im2col_path(cuda, dtype, H, W):
    """conv1_1 with the im2col built in shared memory vs the im2col kernel + 1x1 tensor-core conv, and vs the fp32 reference.
    The fused kernel adds the bias inside the MMA (two spare K columns of ones x bias split into bf16 hi + lo, ~2^-17
    relative), the un-fused path adds the fp32 bias in the epilogue: the bf16 outputs agree except for rare 1-ulp
    rounding flips."""
    from posecnn_b200 import conv
    g = torch.Generator(device="cpu").manual_seed(5)
    B = 2          # W % 4 == 0 with uint8 input takes the staged-patch builder, anything else the per-byte loads
    x = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8).to(cuda) if dtype == torch.uint8 else \
        torch.randn((B, H, W, 3), generator=g).to(cuda)
    mean = (102.9801, 115.9465, 122.7717) if dtype == torch.uint8 else None
    w = (torch.randn((3, 3, 3, 64), generator=g) * 0.2).to(cuda)
    b = torch.randn((64,), generator=g).to(cuda)
    wt = conv.conv1_1_weights_to_tc(w)
    got = conv.conv1_fused(x, wt, b, mean, True)
    want = conv.conv_bf16(conv.im2col_c3(x, mean), wt, b, 1, True)
    torch.cuda.synchronize()
    assert (got == want).float().mean().item() > 0.995
    assert ((got.float() - want.float()).abs() <= 2 ** -7 * want.float().abs().clamp(min=2 ** -6)).all()
    xf = x.float() - (torch.tensor(mean, device=cuda) if mean else 0.0)
    ref = ref_conv(xf.to(torch.bfloat16), w.to(torch.bfloat16), b, True)
    assert ((got.float() - ref).abs() <= 2 ** -7 * ref.abs().clamp(min=1.0)).all()


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 24, 256, 64, 64), (1, 30, 320, 64, 128), (1, 16, 130, 128, 128), (2, 8, 640, 64, 64)])
def test_conv_row_mode(cuda, B, H, W, Cin, Cout):
    """Row mode (two output rows x 128 px per work item, one halo patch shared by the nine taps through row-shifted wgmma
    views; picked automatically for Cin, Cout <= 128 and W >= 128) must agree bit for bit with the 8x16-tile kernel
    (explicit block_n), with and without the fused max pool, and with the fp32 reference."""
    from posecnn_b200 import conv
    g = torch.Generator(device="cpu").manual_seed(321 + W)
    x = torch.randn((B, H, W, Cin), generator=g).to(torch.bfloat16).to(cuda)
    wf = (torch.randn((3, 3, Cin, Cout), generator=g) * (2.0 / (9 * Cin)) ** 0.5).to(torch.bfloat16).to(cuda)
    w = conv.hwio_to_tc(wf.float())
    bias = torch.randn((Cout,), generator=g).to(cuda)
    tile = conv.conv_bf16(x, w, bias, 3, True, Cout)       # explicit N tile -> 8x16-tile kernel
    row = conv.conv_bf16(x, w, bias, 3, True, 0)           # automatic -> row mode
    torch.cuda.synchronize()
    want = ref_conv(x, wf, bias, True)
    assert ((row.float() - want).abs() <= 2 ** -7 * want.abs().clamp(min=1.0)).all()
    if Cin == 64 and Cout == 128:
        assert torch.equal(row, tile)            # same accumulation order -> bit identical
    else:                                        # chunk-outer (Cin = 128) or patch-row-outer (merged two-row MMAs, Cout = 64)
        assert ((row.float() - tile.float()).abs() <= 2 ** -7 * want.abs().clamp(min=1.0)).all()    # order: fp32 rounding only
    rowp = conv.conv_pool_bf16(x, w, bias, 3, True, 0)
    tilep = conv.conv_pool_bf16(x, w, bias, 3, True, Cout)
    torch.cuda.synchronize()
    assert torch.equal(rowp, conv.maxpool2x2(row))
    if Cin == 64 and Cout == 128:
        assert torch.equal(rowp, tilep)


# ---------------------------------------------------------------------------------------------------------------------
# Exact tests at network shapes (tests/util.py: integer operands make every fp32 sum exact in any order, so the bf16 output
# must equal the float64 reference rounded to bf16, bit for bit).  The batch of every case is the smallest that gives each
# persistent CTA at least three work items: the tile loop, the producer running ahead into the next tile, the reuse of the
# epilogue staging buffers and the row mode's resident weights all run.  Shapes are those of a 480 x 640 input.
# ---------------------------------------------------------------------------------------------------------------------
def _network_conv_cases(H=480, W=640):
    """(id, H, W, Cin, Cout, k, pool, dgrad) of every tensor-core convolution of the network and of its training step."""
    from posecnn_b200.networks.vgg16_convs import VGG_CFG
    cases, h, w = [], H, W
    for i, item in enumerate(VGG_CFG):
        if isinstance(item, str):
            h, w = h // 2, w // 2
            continue
        name, ci, co = item
        if name == "conv1_1":                                 # Cin = 3: conv1_fused, below
            continue
        cases.append((name, h, w, ci, co, 3, False, False))   # conv_bf16, as the training step runs every layer
        pooled = i + 1 < len(VGG_CFG) and isinstance(VGG_CFG[i + 1], str) and name not in ("conv4_3", "conv5_3")
        if pooled:                                            # conv_pool_bf16, as inference runs conv1_2, conv2_2, conv3_3
            cases.append((name + "+pool", h, w, ci, co, 3, True, False))
        if ci != co:                                          # input gradient: channels swapped, flipped weights
            cases.append((name + "_dgrad", h, w, co, ci, 3, False, True))
    h4, w4 = H // 8, W // 8
    cases += [("score_conv4", h4, w4, 512, 64, 1, False, False), ("score_conv5", h4 // 2, w4 // 2, 512, 64, 1, False, False),
              ("vertex_folded", h4, w4, 512, 128, 1, False, False),
              ("score_conv4_dgrad", h4, w4, 64, 512, 1, False, True), ("score_conv4_vertex_dgrad", h4, w4, 128, 512, 1, False, True)]
    return cases


def _assert_bits(got, want, what):
    bad = got.view(torch.int16) != want.view(torch.int16)
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outputs differ; first at {idx}: "
                             f"got {got[tuple(idx)].item()} want {want[tuple(idx)].item()}")


_CASES = _network_conv_cases()


@pytest.mark.parametrize("name,H,W,Cin,Cout,k,pool,dgrad", _CASES, ids=[c[0] for c in _CASES])
def test_conv_exact_at_network_shapes(cuda, name, H, W, Cin, Cout, k, pool, dgrad):
    from posecnn_b200 import conv
    from tests.util import conv_batch_for_coverage, int_operands, ref_conv_dgrad_exact, ref_conv_exact
    B, plan = conv_batch_for_coverage(H, W, Cin, Cout, k, pool=pool)
    print(f"{name}: B={B} {plan['kernel']} BN={plan['bn']} tile={plan['tile']} items={plan['items']} grid={plan['grid']} "
          f"-> {plan['per_cta']} items per CTA")
    assert plan["per_cta"] >= 3
    g = torch.Generator().manual_seed(H * 7 + Cin + 3 * Cout + k)
    x = int_operands((B, H, W, Cin), -2, 2, g)
    # forward: HWIO [k, k, Cin, Cout]; input gradient: the forward layer's HWIO [k, k, Cout, Cin] (it maps Cout -> Cin channels)
    w = int_operands((k, k, Cout, Cin) if dgrad else (k, k, Cin, Cout), -2, 2, g)
    bias = int_operands((Cout,), -8, 8, g)
    xd, wd, bd = x.to(cuda), w.to(cuda), bias.to(cuda)
    w_tc = conv.hwio_to_tc_dgrad(wd) if dgrad else conv.hwio_to_tc(wd)
    lin = (ref_conv_dgrad_exact(xd, wd) + bd.double()) if dgrad else ref_conv_exact(xd, wd, bd, False)
    xb = xd.to(torch.bfloat16)
    for relu in (True, False):
        want = lin.clamp(min=0) if relu else lin
        if pool:
            want = torch.nn.functional.max_pool2d(want.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
            got = conv.conv_pool_bf16(xb, w_tc, bd, k, relu)
        else:
            got = conv.conv_bf16(xb, w_tc, bd, k, relu)
        torch.cuda.synchronize()
        _assert_bits(got, want.float().to(torch.bfloat16).contiguous(), f"{name} relu={relu}")
    del lin, want, got


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_conv1_fused_exact_480x640(cuda, dtype):
    """conv1_1 at 480 x 640, batch 2 (4,800 tiles, 36 per CTA): every builder group, both patch buffers of each group and
    both consumer warpgroups run.  uint8 input with integer means (the staged fast path: W % 4 == 0) makes byte - mean an
    integer of magnitude <= 255, exact in bf16, and an integer bias splits into hi + lo with lo = 0: bit-exact output."""
    from posecnn_b200 import conv
    from tests.util import int_operands, num_sms, ref_conv_exact
    B, H, W = 2, 480, 640
    tiles = B * (H // 8) * (W // 16)
    per_cta = tiles // min(tiles, num_sms())
    print(f"conv1_1 {dtype}: {tiles} tiles, {per_cta} per CTA")
    assert per_cta >= 2 * 4                      # four builder groups x two patch buffers
    g = torch.Generator().manual_seed(17)
    if dtype == torch.uint8:
        mean = (103.0, 116.0, 123.0)
        x = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
        xf = x.float() - torch.tensor(mean)
    else:
        mean = None
        x = int_operands((B, H, W, 3), -255, 255, g)
        xf = x
    w = int_operands((3, 3, 3, 64), -2, 2, g)
    bias = int_operands((64,), -8, 8, g)
    wt = conv.conv1_1_weights_to_tc(w.to(cuda))
    lin = ref_conv_exact(xf.to(cuda), w.to(cuda), bias.to(cuda), False)
    for relu in (True, False):
        got = conv.conv1_fused(x.to(cuda), wt, bias.to(cuda), mean, relu)
        torch.cuda.synchronize()
        want = (lin.clamp(min=0) if relu else lin).float().to(torch.bfloat16)
        _assert_bits(got, want, f"conv1_1 {dtype} relu={relu}")
