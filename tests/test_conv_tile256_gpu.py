"""The 256-pixel tile of k_conv_tc (16 x 16 pixels = two 8 x 16 halves, BN = 128), which the dispatcher picks for the 3x3
convolutions with Cin <= 128 and Cout = 128 (conv2_1, conv2_2 (+ pool2), conv2_2's input gradient).

* Against the 128-pixel tile (explicit block_n = 128): bit-identical wherever the two sum in the same order, that is for
  Cin = 64 (one 64-channel chunk) and for maps with odd H or W < 128 (tap-outer, as the 128-pixel tile); within 2 bf16 ulps
  of the fp32 reference for Cin = 128 on maps with even H and W >= 128 (chunk-outer, the order of the row mode these shapes
  ran in before).  Ragged maps put the second half of a tile, or a whole tile, partly or wholly outside the image.
* Exact integer operands at the network's conv2_x shapes (240 x 320), with a batch that gives every persistent CTA at
  least three 256-pixel tiles."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False


def ref_conv(x_bf16, w_hwio_bf16, bias, relu):
    y = F.conv2d(x_bf16.float().permute(0, 3, 1, 2), w_hwio_bf16.float().permute(3, 2, 0, 1), bias, padding=1)
    if relu:
        y = F.relu(y)
    return y.permute(0, 2, 3, 1).contiguous()


def tile256_plan(B, H, W, sms):
    """Work items (256-pixel tiles; one N tile) and grid of a Cout = 128 call."""
    items = B * math.ceil(H / 16) * math.ceil(W / 16)
    return items, min(items, sms)


@pytest.mark.parametrize("B,H,W", [(1, 240, 320), (2, 30, 44), (3, 37, 53), (2, 38, 136)])
@pytest.mark.parametrize("Cin", [64, 128])
def test_tile256_vs_tile128(cuda, B, H, W, Cin):
    from posecnn_b200 import conv
    same_order = Cin == 64 or H % 2 == 1 or W < 128
    g = torch.Generator(device="cpu").manual_seed(4096 + H * W + Cin)
    x = torch.randn((B, H, W, Cin), generator=g).to(torch.bfloat16).to(cuda)
    wf = (torch.randn((3, 3, Cin, 128), generator=g) * (2.0 / (9 * Cin)) ** 0.5).to(torch.bfloat16).to(cuda)
    w = conv.hwio_to_tc(wf.float())
    bias = torch.randn((128,), generator=g).to(cuda)
    for relu in (True, False):
        auto = conv.conv_bf16(x, w, bias, 3, relu)           # 256-pixel tile
        tile = conv.conv_bf16(x, w, bias, 3, relu, 128)      # 128-pixel tile, explicit N tile
        torch.cuda.synchronize()
        want = ref_conv(x, wf, bias, relu)
        tol = 2 ** -7 * want.abs().clamp(min=1.0)            # 2 bf16 ulps
        assert ((auto.float() - want).abs() <= tol).all(), f"relu={relu}: max err {(auto.float() - want).abs().max().item():.4g}"
        if same_order:
            assert torch.equal(auto, tile), f"relu={relu}"
        else:
            assert ((auto.float() - tile.float()).abs() <= tol).all(), f"relu={relu}"
        if H % 2 == 0 and W % 2 == 0:
            autop = conv.conv_pool_bf16(x, w, bias, 3, relu)
            tilep = conv.conv_pool_bf16(x, w, bias, 3, relu, 128)
            torch.cuda.synchronize()
            assert torch.equal(autop, conv.maxpool2x2(auto)), f"relu={relu}"
            if same_order:
                assert torch.equal(autop, tilep), f"relu={relu}"


def _assert_bits(got, want, what):
    bad = got.view(torch.int16) != want.view(torch.int16)
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outputs differ; first at {idx}: "
                             f"got {got[tuple(idx)].item()} want {want[tuple(idx)].item()}")


@pytest.mark.parametrize("name,Cin,pool,dgrad", [("conv2_1", 64, False, False), ("conv2_2", 128, False, False),
                                                 ("conv2_2+pool", 128, True, False), ("conv2_2_dgrad", 128, False, True)])
def test_tile256_exact_at_network_shapes(cuda, name, Cin, pool, dgrad):
    from posecnn_b200 import conv
    from tests.util import int_operands, num_sms, ref_conv_dgrad_exact, ref_conv_exact
    B, H, W, Cout = 2, 240, 320, 128
    items, grid = tile256_plan(B, H, W, num_sms())
    print(f"{name}: B={B} 256-pixel tiles={items} grid={grid} -> {items // grid} per CTA")
    assert items // grid >= 3
    g = torch.Generator().manual_seed(H * 11 + Cin + 5 * Cout + (1 if dgrad else 0))
    x = int_operands((B, H, W, Cin), -2, 2, g)
    w = int_operands((3, 3, Cout, Cin) if dgrad else (3, 3, Cin, Cout), -2, 2, g)
    bias = int_operands((Cout,), -8, 8, g)
    xd, wd, bd = x.to(cuda), w.to(cuda), bias.to(cuda)
    w_tc = conv.hwio_to_tc_dgrad(wd) if dgrad else conv.hwio_to_tc(wd)
    lin = (ref_conv_dgrad_exact(xd, wd) + bd.double()) if dgrad else ref_conv_exact(xd, wd, bd, False)
    xb = xd.to(torch.bfloat16)
    for relu in (True, False):
        want = lin.clamp(min=0) if relu else lin
        if pool:
            want = F.max_pool2d(want.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
            got = conv.conv_pool_bf16(xb, w_tc, bd, 3, relu)
        else:
            got = conv.conv_bf16(xb, w_tc, bd, 3, relu)
        torch.cuda.synchronize()
        _assert_bits(got, want.float().to(torch.bfloat16).contiguous(), f"{name} relu={relu}")
