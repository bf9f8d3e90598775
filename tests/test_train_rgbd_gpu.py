"""The RGB-D training step (posecnn_b200/train.py with input_format='RGBD', the graph of lib/networks/vgg16_convs.py:79-212 with the
depth trunk conv1_1_p .. conv5_3_p of :99-117 and the concat heads of :119-126), and the kernels it adds: the depth-blob im2col of
conv1_1_p's weight gradient and the 1024-channel score_conv4 / score_conv5 GEMMs.  The whole step is compared with torch fp32
autograd of the two-trunk graph built on oracle/ref_network.py, in the 16-bit-rounded and the pure fp32 form, as
tests/test_train_step_gpu.py does for the colour network."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle
from posecnn_b200 import synth
from tests import ref_network as R
from tests.test_train_step_gpu import _ste, ad_loss_torch, rel_l2, to_tf_grad

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
MEANS = (102.9801, 115.9465, 122.7717)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def depth_blob_np(depth_mm):
    """The depth blob of lib/fcn/test.py:70-76 in numpy float32: clip(d / 2000, 0, 1) * 255 tiled x3 - PIXEL_MEANS -> [B,H,W,3]."""
    d = np.asarray(depth_mm, np.float32)
    g = np.clip(d / np.float32(2000.0), np.float32(0.0), np.float32(1.0)) * np.float32(255.0)
    return (g[..., None] - np.asarray(MEANS, np.float32)).astype(np.float32)


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


def _bits(t):
    return t.contiguous().view(torch.int16)


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
    bad = _bits(got) != _bits(want)
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} differ; first at {bad.nonzero()[0].tolist()}"
    assert torch.equal(_bits(got), _bits(via_blob))


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
        bad = _bits(got) != _bits(want)
        assert not bool(bad.any()), f"relu={relu}: {int(bad.sum())} of {bad.numel()} outputs differ"


# ---------------------------------------------------------------------------------------------------------------------
# 4-5. the whole step
# ---------------------------------------------------------------------------------------------------------------------
def make_problem_rgbd(cuda, B=2, H=64, W=96, C=6, seed=0):
    """make_problem of tests/test_train_step_gpu.py for the RGB-D network, plus a depth image in millimetres (synth depth
    x 1000, as bench.py --workload rgbd feeds it) with a clipped band above 2000 mm and a band of zeros."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(input_format="RGBD", num_classes=C, device=cuda, is_train=True, fold_vertex_head=False).init_random(seed=seed, bias_std=0.02)
    net.params["score/weights"] *= 0.02
    net.params["vertex_pred/weights"] *= 0.02
    net.params["fc8/weights"] *= 0.01
    net.prepare()
    rgb, depth = synth.make_images(B, H, W, seed=3)
    dm = (depth * 1000.0).astype(np.float32)
    dm[:, :8] = 2600.0
    dm[:, -4:] = 0.0
    sc = synth.make_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=3, seed=11, min_pixels=200)
    centers = np.zeros((B, C, 3), np.float32)
    for (b, cls, cx, cy, z) in sc["centers"]:
        centers[b, cls] = (cx, cy, z)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    pts = synth.make_model_points(C, 300)
    return (net, T(rgb), T(dm), T(depth_blob_np(dm)), T(sc["label"]), T(centers), T(sc["meta"].reshape(B, 48)), T(sc["extents"]), T(sc["gt"]),
            T(pts), torch.zeros(C, device=cuda))


def reference_grads_rgbd(net, A, data, blob, gt, centers, targets, weights, points, vertex_w, w_inside, margin, sim16):
    """torch fp32 autograd of the two-trunk graph; ROI pooling gathers at OUR arg-max positions.  sim16 as in
    tests/test_train_step_gpu.py: this implementation's op order with every stored activation rounded where our kernels round it."""
    P = {k: v.detach().clone().requires_grad_(True) for k, v in net.params.items()}
    C = net.num_classes
    bf, hf = torch.bfloat16, torch.float16
    r16 = (lambda y: _ste(y, bf)) if sim16 else (lambda y: y)
    rh = (lambda y: _ste(y, hf)) if sim16 else (lambda y: y)
    W = (lambda w: _ste(w, bf)) if sim16 else (lambda w: w)
    Wh = (lambda w: _ste(w, hf)) if sim16 else (lambda w: w)
    x = (data.float() - torch.tensor(MEANS, device=data.device)).permute(0, 3, 1, 2)
    xp = blob.permute(0, 3, 1, 2)

    def trunk16(x, sfx):
        feats = {}
        x = r16(x)
        for item in R.VGG_CFG:
            if isinstance(item, str):
                x = F.max_pool2d(x, 2)
            else:
                x = r16(R.conv(x, W(P[f"{item[0]}{sfx}/weights"]), P[f"{item[0]}{sfx}/biases"]))
                feats[item[0]] = x
        return feats
    f, fp = (trunk16(x, ""), trunk16(xp, "_p")) if sim16 else (R.trunk(P, x), R.trunk(P, xp, "_p"))
    c4, c5 = f["conv4_3"], f["conv5_3"]
    h4, h5 = torch.cat([c4, fp["conv4_3"]], 1), torch.cat([c5, fp["conv5_3"]], 1)          # concat_conv4 / 5, colour first
    s5 = r16(R.conv(h5, W(P["score_conv5/weights"]), P["score_conv5/biases"]))
    s4 = r16(R.conv(h4, W(P["score_conv4/weights"]), P["score_conv4/biases"]))
    v5 = r16(R.conv(c5, W(P["score_conv5_vertex/weights"]), P["score_conv5_vertex/biases"], False))
    v4 = r16(R.conv(c4, W(P["score_conv4_vertex/weights"]), P["score_conv4_vertex/biases"], False))
    if sim16:
        add_s, add_v = r16(s4 + R.deconv(s5, 4, 2)), r16(v4 + R.deconv(v5, 4, 2))
        zs, zv = torch.zeros(C, device=data.device), torch.zeros(3 * C, device=data.device)
        lr_s = r16(R.conv(add_s, W(P["score/weights"]), zs, False))
        lr_v = r16(R.conv(add_v, W(P["vertex_pred/weights"]), zv, False))
        score = torch.relu(R.deconv(lr_s, 16, 8) + P["score/biases"][None, :, None, None])
        vertex = R.deconv(lr_v, 16, 8) + P["vertex_pred/biases"][None, :, None, None]
        prob = F.softmax(score, 1)
    else:
        score, label, prob, vertex = R.heads_from_scores(P, s4, s5, v4, v5)
    B = data.shape[0]
    g = gt.long()
    pg = prob.detach().gather(1, g.clamp(min=0)[:, None])[:, 0]
    sel = (g >= 0) & ((g > 0) | (pg < net.threshold_label))
    logp = F.log_softmax(score, 1).gather(1, g.clamp(min=0)[:, None])[:, 0]
    loss_cls = -(logp * sel).sum() / (sel.sum() + 1e-10)
    vt, vw = oracle.generate_vertex_targets(gt.cpu().numpy(), centers.cpu().numpy(), w_inside)
    vt, vw = torch.from_numpy(vt).to(data.device).permute(0, 3, 1, 2), torch.from_numpy(vw).to(data.device).permute(0, 3, 1, 2)
    diff = vw * (vertex - vt)
    sl1 = torch.where(diff.abs() < 1, 0.5 * diff * diff, diff.abs() - 0.5)
    loss_vertex = sl1.sum() / (vw.sum() + 1e-10)
    rois = A["rois"]
    n = rois.shape[0]

    def pool(feat, arg):                                  # feat NCHW -> [n, 7*7*C] gather at the stored arg-max (image-relative NHWC index)
        fl = feat.permute(0, 2, 3, 1).reshape(B, -1)
        idx = arg.reshape(n, -1).long()
        b = rois[:, 0].long()
        return fl[b[:, None], idx.clamp(min=0)] * (idx >= 0)
    ps = rh(pool(c5, A["a5"]) + pool(c4, A["a4"]))        # RoiPool reads the colour trunk only (vgg16_convs.py:170-176)
    h6 = rh(torch.relu(ps @ Wh(P["fc6/weights"]) + P["fc6/biases"]))
    h7 = rh(torch.relu(h6 @ Wh(P["fc7/weights"]) + P["fc7/biases"]))
    th = torch.tanh(h7 @ Wh(P["fc8/weights"]) + P["fc8/biases"])
    mul = th * weights
    pred = mul / mul.pow(2).sum(1, keepdim=True).clamp(min=1e-12).sqrt()
    loss_pose = ad_loss_torch(pred, targets, weights, points, margin)
    loss = loss_cls + vertex_w * loss_vertex + loss_pose
    loss.backward()
    return P, dict(loss_cls=loss_cls.item(), loss_vertex=(vertex_w * loss_vertex).item(), loss_pose=loss_pose.item(), score=score.detach(),
                   vertex=vertex.detach())


def _limits(name):
    """(16-bit-rounded, pure fp32) relative-L2 limits of tests/test_train_step_gpu.py for a layer; a `_p` layer gets its colour
    counterpart's."""
    base = name.replace("_p/", "/")
    layer = base.split("/")[0]
    lim16 = 0.2 if base == "conv1_1/w" else (0.15 if layer in ("conv1_1", "conv1_2", "fc6", "fc7", "fc8") else 6e-2)
    lim32 = 0.3 if layer in ("conv1_1", "conv1_2") else (0.15 if layer in ("fc6", "fc7", "fc8") else 0.1)
    return lim16, lim32


def test_rgbd_training_step_matches_fp32_autograd(cuda):
    from posecnn_b200.average_distance_loss import average_distance_loss_op
    from posecnn_b200.train import Trainer
    net, data, dm, blob, gt, centers, meta, ext, gtp, pts, sym = make_problem_rgbd(cuda)
    lr, mu, wd, vw_, wi, margin = 0.01, 0.9, 1e-4, 1.0, 10.0, 0.01
    tr = Trainer(net, lr=lr, momentum=mu, weight_decay=wd, vertex_w=vw_, vertex_w_inside=wi, margin=margin)
    assert tr.master["score_conv4/w"].shape == (net.num_units, 1024) and tr.dg["score_conv4_p"].shape == (512, net.num_units)
    A = tr.forward(data, gt, centers, meta, ext, gtp, pts, sym, depth=dm)
    rows, C = A["rows"], net.num_classes
    assert rows >= 9
    g = torch.Generator().manual_seed(5)            # synthetic quaternion targets on the ROI rows' own classes, as the colour test
    tw, wt = torch.zeros(rows, 4 * C), torch.zeros(rows, 4 * C)
    for r in range(rows):
        c = int(A["rois"][r, 1].item())
        q = torch.randn(4, generator=g); q = q / q.norm()
        tw[r, 4 * c:4 * c + 4] = q; wt[r, 4 * c:4 * c + 4] = 1.0
    tw, wt = tw.to(cuda), wt.to(cuda)
    mul = A["poses_tanh"] * wt
    pred = (mul / mul.pow(2).sum(1, keepdim=True).clamp(min=1e-12).sqrt()).contiguous()
    A["loss_pose_raw"], A["pose_diff"] = average_distance_loss_op.average_distance_loss(pred, tw, wt, pts, sym, margin)
    A["poses_weight"], A["poses_target"] = wt, tw
    grads = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    P, ref = reference_grads_rgbd(net, A, data, blob, gt, centers, tw, wt, pts, vw_, wi, margin, sim16=True)
    Pf, reff = reference_grads_rgbd(net, A, data, blob, gt, centers, tw, wt, pts, vw_, wi, margin, sim16=False)
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
    errs = {}
    for name, gr in grads.items():
        layer, kind = name.split("/")
        key = f"{layer}/{'weights' if kind == 'w' else 'biases'}"
        got = to_tf_grad(tr, name, gr)
        assert got.shape == P[key].grad.shape, name
        e16, e32 = rel_l2(got, P[key].grad), rel_l2(got, Pf[key].grad)
        print(f"grad {name:26s} rel-L2 vs 16-bit-rounded graph {e16:.3e}   vs pure fp32 graph {e32:.3e}   |ref| {P[key].grad.norm().item():.3e}")
        errs[name] = (e16, e32)
    for name, (e16, e32) in errs.items():
        lim16, lim32 = _limits(name)
        assert e16 < lim16, (name, e16, lim16)
        assert e32 < lim32, (name, e32, lim32)
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


def _grads(tr, data, gt, centers, meta, ext, gtp, pts, sym, **kw):
    A = tr.forward(data, gt, centers, meta, ext, gtp, pts, sym, **kw)
    g = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in g.items()}


def test_rgbd_step_depth_and_blob_inputs_agree(cuda):
    """depth= (blob formed in conv1_1_p's loader and in im2col_depth) and data_p= (the numpy float32 blob through the float
    conv1_1 kernel and im2col_c3) feed the same bf16 values to every GEMM: the gradients are bit-identical.  k_up8_bwd sums the
    score / vertex_pred bias gradients with shared-memory float atomics whose order is not fixed, so a tensor that two runs
    with the SAME input already give differently is held to fp32 rounding instead; only those two may be such tensors."""
    from posecnn_b200.train import Trainer
    net, data, dm, blob, gt, centers, meta, ext, gtp, pts, sym = make_problem_rgbd(cuda)
    tr = Trainer(net, lr=0.01)
    args = (data, gt, centers, meta, ext, gtp, pts, sym)
    a = _grads(tr, *args, depth=dm)
    a2 = _grads(tr, *args, depth=dm)
    b = _grads(tr, *args, data_p=blob)
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
TRAIN_WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %r)
from posecnn_b200 import parallel, synth
from posecnn_b200.networks.vgg16_convs import vgg16_convs
from posecnn_b200.train import Trainer
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
B, H, W, C = 4, 64, 96, 6
def problem():
    net = vgg16_convs(input_format="RGBD", num_classes=C, device=dev, is_train=True, fold_vertex_head=False).init_random(seed=0, bias_std=0.02)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02; net.params["fc8/weights"] *= 0.01
    net.prepare()
    return net
rgb, depth = synth.make_images(B, H, W, seed=3)
sc = synth.make_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=3, seed=11, min_pixels=200)
centers = np.zeros((B, C, 3), np.float32)
for (b, cls, cx, cy, z) in sc["centers"]:
    centers[b, cls] = (cx, cy, z)
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
data, gt, cen, meta, ext, gtp = T(rgb), T(sc["label"]), T(centers), T(sc["meta"].reshape(B, 48)), T(sc["extents"]), T(sc["gt"])
dm = T((depth * 1000.0).astype(np.float32))
pts, sym = T(synth.make_model_points(C, 300)), torch.zeros(C, device=dev)
single = Trainer(problem(), lr=0.01, world=1)
ref = single.step(data, gt, cen, meta, ext, gtp, pts, sym, depth=dm)
o, n = parallel.shard_range(B, rank, world)
tr = Trainer(problem(), lr=0.01, world=world)
out = tr.step(data[o:o + n], gt[o:o + n], cen[o:o + n], meta[o:o + n], ext, gtp, pts, sym, batch_global=B, batch_offset=o, depth=dm[o:o + n])
torch.cuda.synchronize()
assert set(out["grads"]) == set(ref["grads"]) == set(tr.master)
worst = 0.0
for name, g in out["grads"].items():
    w = ref["grads"][name]
    e = ((g - w).norm() / w.norm().clamp(min=1e-20)).item()
    worst = max(worst, e)
    assert e < 2e-3, (name, e)
for name in tr.master:
    assert torch.allclose(tr.master[name], single.master[name], rtol=1e-4, atol=1e-6), name
tot = torch.stack([out["loss_cls"][0], out["loss_vertex"][0], out["loss_pose"][0]])
dist.all_reduce(tot)
want = torch.stack([ref["loss_cls"][0], ref["loss_vertex"][0], ref["loss_pose"][0]])
assert torch.allclose(tot, want, rtol=1e-4, atol=1e-6), (tot, want)
dist.barrier()
dist.destroy_process_group()
print("TRAIN_RANK_OK", rank, worst)
''' % ROOT


def test_two_rank_rgbd_training_step_equals_single_gpu(tmp_path):
    """One RGB-D SGD step on image shards over 2 ranks == the step on the whole batch on one GPU (gradients to 2e-3 relative,
    the `_p` gradients all-reduced like every other)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    script = tmp_path / "train_rgbd_worker.py"
    script.write_text(TRAIN_WORKER)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.count("TRAIN_RANK_OK") == 2, (out.stdout[-2000:], out.stderr[-3000:])
