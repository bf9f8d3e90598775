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
    B, p = util.conv_batch_for_coverage(240, 320, 64, 128, 3, sms=132)                # conv2_1: two N tiles, ragged segment
    assert (B, p["kernel"], p["items"], p["per_cta"]) == (1, "row", 720, 5)
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
