"""Shared helpers for the parity tests."""
import math

import numpy as np


def to_np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def assert_hough_rows_equal(got, want, is_train, rtol=1e-4, atol=1e-4, as_set=False):
    """Compare the five Houghvotinggpu outputs.  Integer-valued fields (batch, class, votes,
    domain, weight) exactly; geometry within the stated tolerance (SURVEY.md §8(c))."""
    g = [to_np(x) for x in got]
    w = [to_np(x) for x in want]
    assert g[0].shape == w[0].shape, (g[0].shape, w[0].shape)
    if as_set:
        group = 9 if is_train else 1
        def order(a):
            keys = [tuple(np.round(a[0][i * group][[0, 1]]).astype(int)) +
                    tuple(np.round(a[1][i * group][4:7] * 1e3).astype(int)) for i in range(a[0].shape[0] // group)]
            idx = sorted(range(len(keys)), key=lambda i: keys[i])
            rows = np.concatenate([np.arange(i * group, (i + 1) * group) for i in idx]) if idx else np.arange(0)
            return [x[rows] for x in a]
        if g[0].shape[0] % group == 0:
            g, w = order(g), order(w)
    np.testing.assert_array_equal(g[0][:, [0, 1, 6]], w[0][:, [0, 1, 6]])       # batch, class, votes
    np.testing.assert_allclose(g[0][:, 2:6], w[0][:, 2:6], rtol=rtol, atol=atol)  # box
    np.testing.assert_allclose(g[1], w[1], rtol=rtol, atol=atol)                  # pose
    np.testing.assert_allclose(g[2], w[2], rtol=1e-6, atol=1e-6)                  # target (copied quaternions)
    np.testing.assert_array_equal(g[3], w[3])                                     # weight
    np.testing.assert_array_equal(g[4], w[4])                                     # domain


# ---------------------------------------------------------------------------------------------------------------------
# Exact integer operands.  When every operand is a small integer and sum |a * b| < 2^24 for every output, each bf16 / fp16
# operand and each product is exact, and every fp32 partial sum is an exact integer in ANY order (tensor-core alignment,
# split-K partials, fixed-order finishes).  The kernel's fp32 result is then the true integer, and its bf16 / fp16 store
# rounds that exact value: the output must equal the float64 reference rounded to the same type, bit for bit.  A missing,
# doubled or misplaced tile, K tile, pipeline stage or channel block cannot hide under a tolerance.
# ---------------------------------------------------------------------------------------------------------------------
def int_operands(shape, lo, hi, gen):
    """Seeded float32 tensor of integers drawn uniformly from [lo, hi] (CPU generator, CPU tensor)."""
    import torch
    return torch.randint(lo, hi + 1, tuple(shape), generator=gen).to(torch.float32)


def ref_conv_exact(x_nhwc, w_hwio, bias, relu):
    """SAME / stride-1 convolution + bias (+ ReLU) in float64, NHWC x HWIO -> NHWC; rounded, so the result does not depend
    on the algorithm the backend picks."""
    import torch
    import torch.nn.functional as F
    k = w_hwio.shape[0]
    y = F.conv2d(x_nhwc.double().permute(0, 3, 1, 2), w_hwio.double().permute(3, 2, 0, 1), bias.double(), padding=k // 2)
    if relu:
        y = y.clamp(min=0)
    return y.round().permute(0, 2, 3, 1).contiguous()


def ref_conv_dgrad_exact(dz_nhwc, w_hwio):
    """Input gradient of the SAME / stride-1 convolution with HWIO weights w (x has w.shape[2] channels) in float64:
    torch's adjoint of conv2d, independent of the flipped-weight layout the library feeds its forward kernel."""
    import torch
    k, _, ci, _ = w_hwio.shape
    B, H, W, _ = dz_nhwc.shape
    dx = torch.nn.grad.conv2d_input((B, ci, H, W), w_hwio.double().permute(3, 2, 0, 1), dz_nhwc.double().permute(0, 3, 1, 2),
                                    padding=k // 2)
    return dx.round().permute(0, 2, 3, 1).contiguous()


def ref_wgrad_exact(x_nhwc, dz_nhwc, k):
    """Weight gradient of the SAME / stride-1 convolution in float64, in the tensor-core layout [Cout][tap * Cin + ci]."""
    import torch
    B, H, W, ci = x_nhwc.shape
    co = dz_nhwc.shape[3]
    dw = torch.nn.grad.conv2d_weight(x_nhwc.double().permute(0, 3, 1, 2), (co, ci, k, k), dz_nhwc.double().permute(0, 3, 1, 2),
                                     padding=k // 2)
    return dw.round().permute(0, 2, 3, 1).reshape(co, k * k * ci).contiguous()


def num_sms(sms=None):
    if sms is not None:
        return sms
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# Coverage: how much of a persistent / split-K kernel's looping machinery one call exercises.  These restate the dispatch
# rules of the library (conv_bf16_tc_impl in csrc/conv_tc.cu, plan() in csrc/wgrad_tc.cu, fc_plan in csrc/fc_tc.cu) or read
# the library's own plan through its workspace queries, so that a change to a test shape or to a dispatcher cannot silently
# shrink a case back to one work item per CTA.
# ---------------------------------------------------------------------------------------------------------------------
def conv_plan(B, H, W, Cin, Cout, k, block_n=0, pool=False, sms=None):
    """Work items and grid of one pcnn_conv_bf16_tc / pcnn_conv_pool_bf16_tc call (default N tile, block_n = 0): the 3x3 layers
    with Cin <= 128 run Cout = 128 on the 256-pixel (16 x 16) tile at BN = 128, and Cout = 64 in row mode (two rows x 128 px)."""
    sms = num_sms(sms)
    if block_n == 0 and k == 3 and Cin <= 128 and Cout == 64 and H % 2 == 0 and W >= 128:
        resb = Cin == 64
        items = B * (H // 2) * math.ceil(W / 128)
        return dict(kernel="row_resb" if resb else "row", bn=64, tile=(2, 128), items=items, grid=min(items, sms))
    if block_n == 0 and k == 3 and Cin <= 128 and Cout == 128:
        items = B * math.ceil(H / 16) * math.ceil(W / 16)
        return dict(kernel="tile256", bn=128, tile=(16, 16), items=items, grid=min(items, sms))
    bn = block_n or (256 if Cout % 256 == 0 and k * k * Cin >= 2304 else (128 if Cout % 128 == 0 else 64))
    th, tw = 8, 16
    if not pool and math.ceil(H / 16) * math.ceil(W / 8) < math.ceil(H / 8) * math.ceil(W / 16):
        th, tw = 16, 8
    items = B * math.ceil(H / th) * math.ceil(W / tw) * (Cout // bn)
    return dict(kernel="tile", bn=bn, tile=(th, tw), items=items, grid=min(items, sms))


def conv_batch_for_coverage(H, W, Cin, Cout, k, pool=False, per_cta=3, sms=None):
    """Smallest batch whose every CTA runs at least `per_cta` work items; returns (B, plan)."""
    B = 1
    while True:
        p = conv_plan(B, H, W, Cin, Cout, k, pool=pool, sms=sms)
        if p["items"] // p["grid"] >= per_cta:
            p["per_cta"] = p["items"] // p["grid"]
            return B, p
        B += 1


def wgrad_plan(B, H, W, Cin, Cout, k, lib=None):
    """Split-K plan of one pcnn_conv_wgrad_bf16_tc / pcnn_fc_wgrad_f16_tc call.  The split count is the library's own
    (pcnn_conv_wgrad_workspace_bytes = splits * taps * Cout * Cin floats); the K tiles come from the pixel-box rule
    (64 x 1 for row lists, 16 x 4 for images, 8 x 8 for narrow maps; conv1_2's paired path starts one row above the image)."""
    import ctypes
    if lib is None:
        from posecnn_b200._lib import lib as get_lib
        lib = get_lib()
    nbytes = ctypes.c_size_t(0)
    rc = lib.pcnn_conv_wgrad_workspace_bytes(B, H, W, Cin, Cout, k, ctypes.byref(nbytes))
    assert rc == 0, rc
    per = k * k * Cout * Cin * 4
    assert nbytes.value % per == 0
    splits = nbytes.value // per
    bw, bh = (64, 1) if H == 1 else ((16, 4) if W >= 16 else (8, 8))
    pair64 = Cin == 64 and Cout == 64 and k == 3 and H > 1
    ktiles = B * math.ceil((H + (1 if pair64 else 0)) / bh) * math.ceil(W / bw)
    kps = math.ceil(ktiles / splits)
    assert math.ceil(ktiles / kps) == splits, (ktiles, kps, splits)
    return dict(splits=splits, direct=splits == 1, ktiles=ktiles, ktiles_per_split=kps,
                min_ktiles=ktiles - kps * (splits - 1))


def wgrad_batch_for_coverage(H, W, Cin, Cout, k, min_ktiles=8, lib=None):
    """Smallest batch (for H == 1: row count, in steps of 64) whose every work item runs at least `min_ktiles` K tiles
    (twice the 4-stage ring of k_wgrad_tc); returns (B or rows, plan)."""
    n = 1
    while True:
        p = wgrad_plan(1, 1, n, Cin, Cout, k, lib) if H == 1 else wgrad_plan(n, H, W, Cin, Cout, k, lib)
        if p["min_ktiles"] >= min_ktiles:
            return n, p
        n += 64 if H == 1 else 1


def fc_plan(M, N, K, lib=None):
    """Split-K plan of one pcnn_fc_f16_tc / pcnn_fc_dgrad_f16_tc call, read through pcnn_fc_workspace_bytes
    (splits * M * N floats): splits, 64-wide K chunks per split and the fewest chunks any work item runs."""
    import ctypes
    if lib is None:
        from posecnn_b200._lib import lib as get_lib
        lib = get_lib()
    nbytes = ctypes.c_size_t(0)
    rc = lib.pcnn_fc_workspace_bytes(M, N, K, ctypes.byref(nbytes))
    assert rc == 0, rc
    assert nbytes.value % (M * N * 4) == 0
    splits = nbytes.value // (M * N * 4)
    kchunks = K // 64
    cps = math.ceil(kchunks / splits)
    assert math.ceil(kchunks / cps) == splits, (kchunks, cps, splits)
    return dict(splits=splits, m_tiles=math.ceil(M / 128), chunks_per_split=cps, min_chunks=kchunks - cps * (splits - 1))
