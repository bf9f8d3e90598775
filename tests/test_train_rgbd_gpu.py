"""The RGB-D training step (posecnn_b200/train.py with input_format='RGBD', the graph of lib/networks/vgg16_convs.py:79-212 with the
depth trunk conv1_1_p .. conv5_3_p of :99-117 and the concat heads of :119-126), and the kernels it adds: the depth-blob im2col of
conv1_1_p's weight gradient and the 1024-channel score_conv4 / score_conv5 GEMMs.  The whole step is compared with torch fp32
autograd of the two-trunk graph (tests/train_ref.py reference_grads with depth_blob=), in the 16-bit-rounded and the pure fp32
form, as tests/test_train_step_gpu.py does for the colour network."""
import numpy as np
import pytest
import torch

from tests.train_ref import (MEANS, bits, compare_grads, depth_blob_np, grads_of, make_inputs, make_net, reference_grads, rel_l2,
                             run_two_ranks, synthetic_pose_targets, train_worker)

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def im2col_np(x):
    """[B,H,W,3] f32 -> [B,H,W,64] f32, K = (dy * 3 + dx) * 3 + c (SAME zero padding), columns 27..63 zero."""
    B, H, W, _ = x.shape
    xp = np.zeros((B, H + 2, W + 2, 3), np.float32)
    xp[:, 1:-1, 1:-1] = x
    out = np.zeros((B, H, W, 64), np.float32)
    for dy in range(3):
        for dx in range(3):
            t = dy * 3 + dx
            out[..., 3 * t:3 * t + 3] = xp[:, dy:dy + H, dx:dx + W]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1-2. the depth-blob im2col
# ---------------------------------------------------------------------------------------------------------------------
def _edge_depth(B, H, W, seed):
    """Depths in millimetres over [-500, 2600] with exact 0, exact 2000, negative values and values above the 2000 mm clip."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(-500.0, 2600.0, (B, H, W)).astype(np.float32)
    d[:, ::7, ::5] = 0.0
    d[:, 3::11, 2::9] = 2000.0
    d[:, :, -1] = 2500.0                                 # the last column, at the image border, clipped to 255
    d[:, 0, :] = -1.0                                    # the first row clipped to 0
    return d


@pytest.mark.parametrize("B,H,W", [(2, 37, 133), (1, 16, 128), (3, 9, 20)])
def test_im2col_depth_bit_exact(cuda, B, H, W):
    """Every element equals the numpy float32 blob rounded once to bf16; also equals im2col_c3 (float) of that blob."""
    from posecnn_b200 import conv
    d = _edge_depth(B, H, W, seed=H * W)
    blob = depth_blob_np(d)
    want = torch.from_numpy(im2col_np(blob)).to(torch.bfloat16).to(cuda)
    got = conv.im2col_depth(torch.from_numpy(d).to(cuda), MEANS)
    via_blob = conv.im2col_c3(torch.from_numpy(blob).to(cuda), None)
    torch.cuda.synchronize()
    assert got.shape == (B, H, W, 64)
    bad = bits(got) != bits(want)
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} differ; first at {bad.nonzero()[0].tolist()}"
    assert torch.equal(bits(got), bits(via_blob))


@pytest.mark.parametrize("H,W", [(37, 53), (48, 80), (64, 96)])
def test_conv1_im2col_depth_matches_fused(cuda, H, W):
    """conv_bf16(im2col_depth(d)) against conv1_depth_fused(d): the bound test_conv1_fused_matches_im2col_path uses for colour
    (the fused kernel adds the bias inside the MMA as bf16 hi + lo, the 1x1 path in the fp32 epilogue: rare 1-ulp flips)."""
    from posecnn_b200 import conv
    g = torch.Generator(device="cpu").manual_seed(H + W)
    d = torch.from_numpy(_edge_depth(2, H, W, seed=W)).to(cuda)
    w = (torch.randn((3, 3, 3, 64), generator=g) * 0.2).to(cuda)
    b = torch.randn((64,), generator=g).to(cuda)
    wt = conv.conv1_1_weights_to_tc(w)
    for relu in (True, False):
        got = conv.conv1_depth_fused(d, wt, b, MEANS, relu)
        want = conv.conv_bf16(conv.im2col_depth(d, MEANS), wt, b, 1, relu)
        torch.cuda.synchronize()
        same = (got == want).float().mean().item()
        print(f"{H}x{W} relu={relu}: {same:.5f} identical")
        assert same > 0.995
        assert ((got.float() - want.float()).abs() <= 2 ** -7 * want.float().abs().clamp(min=2 ** -6)).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3. exact integer tests at the new GEMM shapes (tests/util.py): Cin = 1024 at 480 x 640's score_conv4 / score_conv5 maps
# ---------------------------------------------------------------------------------------------------------------------
_CIN1024 = [("score_conv4", 60, 80), ("score_conv5", 30, 40)]


@pytest.mark.parametrize("name,H,W", _CIN1024, ids=[c[0] for c in _CIN1024])
def test_wgrad_exact_cin1024(cuda, name, H, W):
    from posecnn_b200 import backward
    from tests.util import int_operands, ref_wgrad_exact, wgrad_batch_for_coverage
    B, plan = wgrad_batch_for_coverage(H, W, 1024, 64, 1)
    print(f"{name} concat wgrad: B={B} splits={plan['splits']} ktiles={plan['ktiles']} -> {plan['min_ktiles']}..{plan['ktiles_per_split']} "
          f"K tiles per item")
    assert plan["min_ktiles"] >= 8
    g = torch.Generator().manual_seed(H + 1024)
    x = int_operands((B, H, W, 1024), -1, 1, g).to(torch.bfloat16).to(cuda)
    dz = int_operands((B, H, W, 64), -1, 1, g).to(torch.bfloat16).to(cuda)
    want = ref_wgrad_exact(x, dz, 1).float()
    got = backward.conv_wgrad(x, dz, 1)
    torch.cuda.synchronize()
    bad = got != want
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} gradients differ; first at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("name,H,W", _CIN1024, ids=[c[0] for c in _CIN1024])
def test_conv_exact_cin1024(cuda, name, H, W):
    from posecnn_b200 import conv
    from tests.util import conv_batch_for_coverage, int_operands, ref_conv_exact
    B, plan = conv_batch_for_coverage(H, W, 1024, 64, 1)
    print(f"{name} concat 1x1: B={B} {plan['kernel']} BN={plan['bn']} tile={plan['tile']} items={plan['items']} grid={plan['grid']} "
          f"-> {plan['per_cta']} items per CTA")
    assert plan["per_cta"] >= 3
    g = torch.Generator().manual_seed(W + 1024)
    x = int_operands((B, H, W, 1024), -2, 2, g)
    w = int_operands((1, 1, 1024, 64), -2, 2, g)
    bias = int_operands((64,), -8, 8, g)
    xd, wd, bd = x.to(cuda), w.to(cuda), bias.to(cuda)
    lin = ref_conv_exact(xd, wd, bd, False)
    for relu in (True, False):
        got = conv.conv_bf16(xd.to(torch.bfloat16), conv.hwio_to_tc(wd), bd, 1, relu)
        torch.cuda.synchronize()
        want = (lin.clamp(min=0) if relu else lin).float().to(torch.bfloat16)
        bad = bits(got) != bits(want)
        assert not bool(bad.any()), f"relu={relu}: {int(bad.sum())} of {bad.numel()} outputs differ"


# ---------------------------------------------------------------------------------------------------------------------
# 4-5. the whole step
# ---------------------------------------------------------------------------------------------------------------------
def rgbd_inputs(cuda):
    """make_inputs' labelled batch and its depth image with a clipped band above 2000 mm and a band of zeros, and that depth's
    numpy float32 blob."""
    args, _, dm = make_inputs(cuda)
    dm[:, :8] = 2600.0
    dm[:, -4:] = 0.0
    return args, dm, torch.from_numpy(depth_blob_np(dm.cpu().numpy())).to(cuda)


def test_rgbd_training_step_matches_fp32_autograd(cuda):
    from posecnn_b200.train import Trainer
    net = make_net(cuda, "RGBD")
    args, dm, blob = rgbd_inputs(cuda)
    data, gt, centers, meta, ext, gtp, pts, sym = args
    lr, mu, wd, vw_, wi, margin = 0.01, 0.9, 1e-4, 1.0, 10.0, 0.01
    tr = Trainer(net, lr=lr, momentum=mu, weight_decay=wd, vertex_w=vw_, vertex_w_inside=wi, margin=margin)
    assert tr.master["score_conv4/w"].shape == (net.num_units, 1024) and tr.dg["score_conv4_p"].shape == (512, net.num_units)
    A = tr.forward(data, gt, centers, meta, ext, gtp, pts, sym, depth=dm)
    assert A["rows"] >= 9
    tw, wt = synthetic_pose_targets(A, pts, sym, margin)
    grads = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    P, ref = reference_grads(net, A, args, tw, wt, True, vw_, wi, margin, depth_blob=blob)
    Pf, reff = reference_grads(net, A, args, tw, wt, False, vw_, wi, margin, depth_blob=blob)
    e = [rel_l2(A["score"].permute(0, 3, 1, 2), ref["score"]), rel_l2(tr.dense_vertex_pred(A).permute(0, 3, 1, 2), ref["vertex"]),
         rel_l2(A["score"].permute(0, 3, 1, 2), reff["score"]), rel_l2(tr.dense_vertex_pred(A).permute(0, 3, 1, 2), reff["vertex"])]
    print("forward score / vertex rel-L2 vs 16-bit-rounded graph %.3e %.3e, vs pure fp32 graph %.3e %.3e" % tuple(e))
    assert e[0] < 5e-3 and e[1] < 5e-3 and e[2] < 3e-2 and e[3] < 3e-2
    for r_ in (ref, reff):
        assert abs(A["cls_out"][0].item() - r_["loss_cls"]) < 3e-2 * max(1.0, abs(r_["loss_cls"]))
        assert abs(vw_ * A["vtx_out"][0].item() - r_["loss_vertex"]) < 3e-2 * max(1.0, abs(r_["loss_vertex"]))
        assert abs(A["loss_pose"].item() - r_["loss_pose"]) < 3e-2 * max(1e-3, abs(r_["loss_pose"]))
    assert set(grads) == set(tr.master)
    assert sum(1 for k in grads if k.split("/")[0].endswith("_p")) == 26
    compare_grads(tr, grads, P, Pf, list(grads))
    # the update: accum = grad + wd * w (first step), w -= lr * accum; 16-bit copies and the padded conv1_1_p tile refreshed
    before = {k: v.clone() for k, v in tr.master.items()}
    tr.update(grads)
    for name in ("conv3_2_p/w", "conv1_1_p/w", "conv5_3_p/b", "score_conv4/w", "score_conv5/w", "conv3_2/w", "fc7/w", "score/b"):
        want = before[name] - lr * (grads[name] + wd * before[name])
        assert torch.allclose(tr.master[name], want, rtol=1e-5, atol=1e-7), name
    assert torch.equal(tr.tc["conv3_2_p/w"], tr.master["conv3_2_p/w"].to(torch.bfloat16))
    assert torch.equal(tr.tc["score_conv4/w"], tr.master["score_conv4/w"].to(torch.bfloat16))
    assert torch.equal(tr.conv1_tc_p[:, :27], tr.master["conv1_1_p/w"].to(torch.bfloat16))
    # a second full step runs (momentum path); exported params feed the inference network's RGB-D forward
    out = tr.step(data, gt, centers, meta, ext, gtp, pts, sym, depth=dm)
    assert torch.isfinite(out["loss"]).all()
    tr.export_params()
    assert torch.allclose(net.params["conv3_2_p/weights"].permute(3, 0, 1, 2).reshape(256, -1), tr.master["conv3_2_p/w"])
    assert torch.equal(net.params["score_conv4/weights"].reshape(1024, -1).t(), tr.master["score_conv4/w"])
    assert torch.equal(net._tc["conv1_1_p/weights"], tr.conv1_tc_p)      # the inference copy is the trained conv1_1_p tile
    L = net.forward(data, meta, ext, poses=gtp, depth=dm, want_score=True)
    torch.cuda.synchronize()
    assert torch.isfinite(L["score"]).all() and L["rois"].shape[0] >= 1


def test_rgbd_step_depth_and_blob_inputs_agree(cuda):
    """depth= (blob formed in conv1_1_p's loader and in im2col_depth) and data_p= (the numpy float32 blob through the float
    conv1_1 kernel and im2col_c3) feed the same bf16 values to every GEMM: the gradients are bit-identical.  Run-to-run
    bit-identity is not required of the score / vertex_pred bias gradients (sums over every pixel of the batch): a tensor that two
    runs with the SAME input already give differently is held to fp32 rounding instead; only those two may be such tensors."""
    from posecnn_b200.train import Trainer
    args, dm, blob = rgbd_inputs(cuda)
    tr = Trainer(make_net(cuda, "RGBD"), lr=0.01)
    a = grads_of(tr, args, depth=dm)
    a2 = grads_of(tr, args, depth=dm)
    b = grads_of(tr, args, data_p=blob)
    assert set(a) == set(b) == set(tr.master)
    unfixed = {k for k in a if not torch.equal(a[k], a2[k])}
    print("tensors that differ between two runs of one input form:", sorted(unfixed))
    assert unfixed <= {"score/b", "vertex_pred/b"}
    for k in a:
        if k in unfixed:
            assert torch.allclose(a[k], b[k], rtol=1e-5, atol=1e-9), k
        else:
            assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# 8. two ranks
# ---------------------------------------------------------------------------------------------------------------------
def test_two_rank_rgbd_training_step_equals_single_gpu(tmp_path):
    """One RGB-D SGD step on image shards over 2 ranks == the step on the whole batch on one GPU (gradients to 2e-3 relative,
    the `_p` gradients all-reduced like every other)."""
    run_two_ranks(tmp_path, train_worker("RGBD"))
