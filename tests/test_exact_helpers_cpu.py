"""CPU rehearsal of the exact-integer test helpers (tests/util.py): the float64 references agree with an fp32 computation on
integer operands (exact in any order), and the coverage helpers reproduce the dispatch plans the GPU tests rely on."""
import torch
import torch.nn.functional as F

from tests import util


def test_references_on_integer_operands():
    g = torch.Generator().manual_seed(0)
    for k in (1, 3):
        x = util.int_operands((2, 9, 11, 8), -2, 2, g)
        w = util.int_operands((k, k, 8, 6), -2, 2, g)
        b = util.int_operands((6,), -8, 8, g)
        y32 = F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, padding=k // 2).permute(0, 2, 3, 1)
        assert torch.equal(util.ref_conv_exact(x, w, b, False), y32.double())
        assert torch.equal(util.ref_conv_exact(x, w, b, True), y32.clamp(min=0).double())
        dz = util.int_operands((2, 9, 11, 6), -1, 1, g)
        xr = x.clone().requires_grad_(True)
        wr = w.permute(3, 2, 0, 1).contiguous().requires_grad_(True)
        F.conv2d(xr.permute(0, 3, 1, 2), wr, padding=k // 2).backward(dz.permute(0, 3, 1, 2))
        assert torch.equal(util.ref_conv_dgrad_exact(dz, w), xr.grad.double())
        assert torch.equal(util.ref_wgrad_exact(x, dz, k), wr.grad.permute(0, 2, 3, 1).reshape(6, k * k * 8).double())


def test_first_max_route_reference():
    from tests.test_backward_gpu import first_max_route
    g = torch.Generator().manual_seed(1)
    y = torch.relu(util.int_operands((1, 4, 6, 8), -1, 2, g))
    gp = util.int_operands((1, 2, 3, 8), 1, 3, g)
    want = torch.zeros_like(y)
    for i in range(2):
        for j in range(3):
            for c in range(8):
                win = [y[0, 2 * i, 2 * j, c], y[0, 2 * i, 2 * j + 1, c], y[0, 2 * i + 1, 2 * j, c], y[0, 2 * i + 1, 2 * j + 1, c]]
                best = max(range(4), key=lambda q: (win[q], -q))        # first maximum in raster order
                if win[best] > 0:
                    want[0, 2 * i + best // 2, 2 * j + best % 2, c] = gp[0, i, j, c]
    assert torch.equal(first_max_route(gp, y).float(), want)


def test_coverage_helpers(native_lib):
    B, p = util.conv_batch_for_coverage(480, 640, 64, 64, 3, sms=132)                 # conv1_2: RESB row mode, 5 segments
    assert (B, p["kernel"], p["items"], p["per_cta"]) == (1, "row_resb", 1200, 9)
    B, p = util.conv_batch_for_coverage(240, 320, 64, 128, 3, sms=132)                # conv2_1: 256-pixel tile, BN = 128
    assert (B, p["kernel"], p["items"], p["per_cta"]) == (2, "tile256", 600, 4)
    B, p = util.conv_batch_for_coverage(30, 40, 512, 512, 3, sms=132)                 # conv5: 16 x 8 tiles
    assert (B, p["tile"], p["bn"], p["per_cta"]) == (20, (16, 8), 256, 3)
    B, p = util.conv_batch_for_coverage(120, 160, 256, 256, 3, pool=True, sms=132)    # fused pool: always 8 x 16
    assert (B, p["tile"], p["per_cta"]) == (3, (8, 16), 3)
    p = util.wgrad_plan(1, 480, 640, 64, 64, 3, native_lib)                             # conv1_2: paired path, row -1 origin
    assert p["ktiles"] == 121 * 40 and p["min_ktiles"] >= 8
    assert util.wgrad_plan(1, 1, 600, 25088, 4096, 1, native_lib) == dict(splits=1, direct=True, ktiles=10, ktiles_per_split=10,
                                                                          min_ktiles=10)
    rows, p = util.wgrad_batch_for_coverage(1, 1, 192, 4096, 1, lib=native_lib)
    assert p["min_ktiles"] >= 8 and rows % 64 == 1
    assert util.fc_plan(600, 4096, 25088, native_lib)["splits"] == 1
    assert util.fc_plan(600, 128, 4096, native_lib)["splits"] == 16


def test_conv_plan_follows_the_dispatcher():
    """conv_bf16_tc_impl (csrc/conv_tc.cu) runs the 3x3, Cin <= 128 layers with Cout = 128 on the 256-pixel tile (16 x 16,
    BN = 128) and only Cout = 64 in row mode.  At 132 SMs every conv2 case of test_conv_exact_at_network_shapes therefore needs
    batch 2 for three work items per CTA; the 720 x 960 shapes of test_rescale_gpu.py get there at batch 1."""
    from tests.test_conv_gpu import _network_conv_cases
    for H, W, want_B in ((480, 640, 2), (720, 960, 1)):
        cases = {c[0]: c for c in _network_conv_cases(H, W)}
        for name in ("conv2_1", "conv2_2", "conv2_2+pool"):
            _, h, w, ci, co, k, pool, _ = cases[name]
            B, p = util.conv_batch_for_coverage(h, w, ci, co, k, pool=pool, sms=132)
            assert (p["kernel"], p["tile"], p["bn"]) == ("tile256", (16, 16), 128), (name, p)
            assert p["items"] == B * -(-h // 16) * -(-w // 16) and p["grid"] == 132, (name, p)
            assert (B, p["per_cta"] >= 3) == (want_B, True), (name, H, B, p)
        for name in ("conv1_2", "conv1_2+pool", "conv2_1_dgrad"):                    # Cout = 64: row mode
            _, h, w, ci, co, k, pool, _ = cases[name]
            assert util.conv_plan(1, h, w, ci, co, k, pool=pool, sms=132)["kernel"] in ("row", "row_resb"), name
        assert util.conv_plan(1, 240, 320, 64, 128, 3, block_n=128, sms=132)["tile"] == (8, 16)   # explicit N tile: 128 pixels
