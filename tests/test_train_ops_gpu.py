"""GPU parity of the training-side target generation and fused losses (SURVEY.md §8(f) rank 3) against the reference's
own _generate_vertex_targets output (tests/golden/vertex_targets.npz) and the numpy restatements of the TF loss graphs."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.golden import cases
from tests.util import to_np

pytestmark = pytest.mark.gpu
T = lambda a, dev: torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def test_vertex_targets_match_reference_golden(cuda):
    from posecnn_b200 import train_ops
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "vertex_targets.npz"))
    label, centers = cases.vertex_target_inputs()
    t, w = train_ops.generate_vertex_targets(T(label, cuda), T(centers, cuda), 10.0)
    np.testing.assert_array_equal(to_np(w), g["weights"])
    got, want = to_np(t), g["targets"]
    # direction components: float64 divide rounded to float32 -- bit exact; log z: double log, <= 1 float32 ulp
    np.testing.assert_array_equal(got[..., 0::3], want[..., 0::3])
    np.testing.assert_array_equal(got[..., 1::3], want[..., 1::3])
    np.testing.assert_allclose(got[..., 2::3], want[..., 2::3], rtol=1.2e-7, atol=0)


def test_vertex_targets_full_size_properties(cuda):
    """640x480x22 at batch 4: unit direction vectors, weights only on labelled pixels of listed classes, equals the oracle."""
    from posecnn_b200 import synth, train_ops
    sc = synth.make_scene(batch=4, height=480, width=640, num_classes=22, seed=99)
    label = sc["label"]
    C = 22
    rng = np.random.default_rng(1)
    centers = np.zeros((4, C, 3), np.float32)
    for b in range(4):
        for c in np.unique(label[b]):
            if c > 0:
                ys, xs = np.where(label[b] == c)
                centers[b, c] = (xs.mean() + rng.normal(), ys.mean() + rng.normal(), rng.uniform(0.5, 1.5))
    t, w = train_ops.generate_vertex_targets(T(label, cuda), T(centers, cuda), 10.0)
    wt, ww = oracle.generate_vertex_targets(label, centers, 10.0)
    np.testing.assert_array_equal(to_np(w), ww)
    np.testing.assert_allclose(to_np(t), wt, rtol=1.2e-7, atol=0)
    tt = to_np(t).reshape(4, 480, 640, C, 3)
    fg = label > 0
    sel = np.take_along_axis(tt, np.maximum(label, 0)[..., None, None].astype(np.int64), axis=3)[..., 0, :]
    n = np.hypot(sel[..., 0], sel[..., 1])[fg]
    assert np.all((np.abs(n - 1) < 1e-5) | (n == 0))


@pytest.mark.parametrize("threshold", [1.0, 0.4])
def test_loss_cross_entropy_hard(cuda, threshold):
    from posecnn_b200 import train_ops
    rng = np.random.default_rng(3)
    B, H, W, C = 2, 48, 64, 22
    logits = rng.standard_normal((B, H, W, C)).astype(np.float32) * 2
    score = logits - np.log(np.exp(logits).sum(3, keepdims=True))          # log-softmax
    prob = np.exp(score).astype(np.float32)
    gt = rng.integers(-1, C, size=(B, H, W)).astype(np.int32)
    want, mask = oracle.loss_cross_entropy_hard(score, prob, gt, threshold)
    loss, count, grad = train_ops.loss_cross_entropy_hard(T(score, cuda), T(prob, cuda), T(gt, cuda), threshold, want_grad=True)
    assert float(count.item()) == mask.sum()                                 # selection: exact
    assert abs(float(loss.item()) - want) <= 1e-5 * abs(want)                # stated tolerance: rel 1e-5 (fp32 result of a double sum)
    np.testing.assert_allclose(to_np(grad), (-mask / (mask.sum() + 1e-10)).astype(np.float32), rtol=1e-6, atol=0)
    # deterministic: bit-identical across launches
    loss2, _ = train_ops.loss_cross_entropy_hard(T(score, cuda), T(prob, cuda), T(gt, cuda), threshold)
    assert float(loss2.item()) == float(loss.item())
    # the fused loss equals the un-fused composition through the Hardlabel op
    from posecnn_b200.hard_label_layer import hard_label_op
    m = hard_label_op.hard_label(T(prob, cuda), T(gt, cuda), threshold)
    comp = -(m.double() * T(score, cuda).double()).sum() / (m.double().sum() + 1e-10)
    assert abs(float(loss.item()) - float(comp.item())) <= 1e-5 * abs(float(comp.item()))


@pytest.mark.parametrize("sigma,n", [(1.0, 4 * 30 * 40 * 66), (3.0, 1001)])
def test_smooth_l1_loss_vertex(cuda, sigma, n):
    from posecnn_b200 import train_ops
    rng = np.random.default_rng(4)
    pred = rng.standard_normal(n).astype(np.float32)
    targ = rng.standard_normal(n).astype(np.float32)
    wgt = np.where(rng.random(n) < 0.2, 10.0, 0.0).astype(np.float32)
    pad = (-n) % 4                                                   # the wrapper needs 16-byte aligned tensors, any length
    want, gwant = oracle.smooth_l1_loss_vertex(pred, targ, wgt, sigma)
    loss, wsum, grad = train_ops.smooth_l1_loss_vertex(T(pred, cuda), T(targ, cuda), T(wgt, cuda), sigma, want_grad=True)
    assert float(wsum.item()) == float(wgt.astype(np.float64).sum())
    assert abs(float(loss.item()) - want) <= 1e-5 * abs(want)
    np.testing.assert_allclose(to_np(grad), gwant, rtol=1e-5, atol=1e-9)
    # gradient check against torch autograd of the reference formula
    p = T(pred, cuda).double().requires_grad_()
    d = T(wgt, cuda).double() * (p - T(targ, cuda).double())
    s2 = sigma ** 2
    sign = (d.abs() < 1.0 / s2).double().detach()
    l = ((d ** 2) * (s2 / 2) * sign + (d.abs() - 0.5 / s2) * (1 - sign)).sum() / (T(wgt, cuda).double().sum() + 1e-10)
    l.backward()
    assert torch.allclose(grad.double(), p.grad, rtol=1e-4, atol=1e-9)


def test_training_loss_heads_compose(cuda):
    """configs[4] shape in miniature (a GPU's share of the batch): is_train network forward -> Hough in train mode
    (9 jittered rows per ROI, quaternion targets from the gt poses) -> RoiPool -> pose head -> the three training losses,
    each against the oracle composition on the network's own intermediate tensors."""
    from posecnn_b200 import synth, train_ops
    from posecnn_b200.networks.vgg16_convs import training_losses, vgg16_convs
    C, B, H, W = 6, 2, 64, 96
    net = vgg16_convs(num_classes=C, device=cuda, is_train=True).init_random(seed=0, bias_std=0.05)
    rgb, _ = synth.make_images(B, H, W, seed=3)
    data = torch.from_numpy(rgb).to(cuda)
    meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)).to(cuda)
    ext = torch.from_numpy(synth.extents_for(C)).to(cuda)
    rng = np.random.default_rng(8)
    gt = np.zeros((2 * (C - 1), 13), np.float32)                      # gt pose rows [batch, cls, (5 unused), qw..qz, t]
    for i in range(gt.shape[0]):
        q = rng.standard_normal(4); q /= np.linalg.norm(q)
        gt[i, 0], gt[i, 1] = i % B, 1 + i // B
        gt[i, 2:6] = (10, 10, 80, 60); gt[i, 6:10] = q; gt[i, 10:13] = (0.0, 0.0, 1.0)
    out = net.forward(data, meta, ext, poses=torch.from_numpy(gt).to(cuda), want_prob=True, want_score=True)
    label = to_np(out["label_2d"])
    u = rng.random(label.shape)                                                         # 10 % ignore, 30 % disagreeing labels
    gt_label = np.where(u < 0.1, -1, np.where(u < 0.4, rng.integers(0, C, label.shape), label)).astype(np.int32)
    centers = np.zeros((B, C, 3), np.float32)
    for b in range(B):
        for c in np.unique(label[b]):
            if c > 0:
                ys, xs = np.where(label[b] == c)
                centers[b, c] = (xs.mean(), ys.mean(), 0.8 + 0.1 * c)
    vt, vw = train_ops.generate_vertex_targets(T(label, cuda), T(centers, cuda), 10.0)
    points = T(synth.make_model_points(C, 200, seed=2), cuda)
    symmetry = torch.zeros((C,), device=cuda); symmetry[2] = 1.0
    losses = training_losses(net, out, T(gt_label, cuda), vt, vw, points, symmetry, vertex_w=1.0)
    # classification: log-softmax of the kernel's own scores, Hardlabel selection
    score = to_np(out["score"]).astype(np.float64)
    logp = score - np.log(np.exp(score - score.max(3, keepdims=True)).sum(3, keepdims=True)) - score.max(3, keepdims=True)
    want_cls, _ = oracle.loss_cross_entropy_hard(logp, to_np(out["prob_normalized"]), gt_label, 1.0)
    assert want_cls > 1e-3 and abs(float(losses["loss_cls"].item()) - want_cls) <= 2e-5 * abs(want_cls)
    want_v, _ = oracle.smooth_l1_loss_vertex(to_np(out["vertex_pred"]), to_np(vt), to_np(vw), 1.0)
    assert abs(float(losses["loss_vertex"].item()) - want_v) <= 1e-5 * abs(want_v)
    # pose: rows come in groups of 9 per ROI in train mode; weights select the gt class quaternion
    assert out["rois"].shape[0] % 9 == 0 and out["poses_weight"].shape == out["poses_tanh"].shape
    pt, pw, ptg = to_np(out["poses_tanh"]), to_np(out["poses_weight"]), to_np(out["poses_target"])
    mul = pt * pw
    pred = mul / np.sqrt(np.maximum((mul ** 2).sum(1, keepdims=True), 1e-12))
    want_p, _ = oracle.average_distance_loss(pred.astype(np.float32), ptg, pw, to_np(points), to_np(symmetry), 0.01)
    assert abs(float(losses["loss_pose"].item()) - float(want_p[0])) <= 1e-4 * max(abs(float(want_p[0])), 1e-6)
    total = float(losses["loss_cls"].item()) + float(losses["loss_vertex"].item()) + float(losses["loss_pose"].item())
    assert abs(float(losses["loss"].item()) - total) <= 1e-5 * abs(total)


def test_vertex_loss_fused_equals_materialised(cuda):
    """The fused vertex loss (labels + centres in, no target / weight tensors) == smooth L1 on the materialised targets,
    forward and gradient, at full frame size."""
    from posecnn_b200 import synth, train_ops
    sc = synth.make_scene(batch=2, height=480, width=640, num_classes=22, seed=77)
    label = sc["label"]
    rng = np.random.default_rng(2)
    centers = np.zeros((2, 22, 3), np.float32)
    for b in range(2):
        for c in np.unique(label[b]):
            if c > 0:
                ys, xs = np.where(label[b] == c)
                centers[b, c] = (xs.mean() + rng.normal(), ys.mean() + rng.normal(), rng.uniform(0.5, 1.5))
    centers[0, int(np.unique(label[0])[1]), 2] = 0.0                  # one labelled class not listed
    pred = T(sc["vertex"], cuda) + 0.3 * torch.randn(sc["vertex"].shape, device=cuda)
    lab, cen = T(label, cuda), T(centers, cuda)
    for sigma in (1.0, 2.5):
        vt, vw = train_ops.generate_vertex_targets(lab, cen, 10.0)
        l0, w0, g0 = train_ops.smooth_l1_loss_vertex(pred, vt, vw, sigma, want_grad=True, upstream=0.7)
        l1, w1, g1 = train_ops.vertex_loss_from_centers(pred, lab, cen, 10.0, sigma, want_grad=True, upstream=0.7)
        assert float(w0.item()) == float(w1.item()) > 0
        assert abs(float(l0.item()) - float(l1.item())) <= 1e-6 * abs(float(l0.item()))
        assert torch.equal(g0, g1)
        want, _ = oracle.smooth_l1_loss_vertex(to_np(pred), to_np(vt), to_np(vw), sigma)
        assert abs(float(l1.item()) - want) <= 1e-5 * abs(want)


def test_multi_instance_vertex_targets_match_reference_golden(cuda):
    """pcnn_vertex_targets_instances_fwd vs the reference function's own output on the multi-instance branch
    (minibatch.py:549-573; tests/golden/vertex_targets_multi.npz): direction components bit-exact, log z to 1 ulp of libm."""
    from posecnn_b200 import train_ops
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "vertex_targets_multi.npz"))
    label, mask, inst = cases.vertex_target_multi_inputs()
    t, w = train_ops.generate_vertex_targets_instances(T(label, cuda), T(mask, cuda), T(inst, cuda), 6, 10.0)
    t, w = t.cpu().numpy(), w.cpu().numpy()
    np.testing.assert_array_equal(w, g["weights"])
    xy = np.ones(t.shape[-1], bool); xy[2::3] = False
    np.testing.assert_array_equal(t[..., xy], g["targets"][..., xy])
    np.testing.assert_allclose(t[..., ~xy], g["targets"][..., ~xy], rtol=2e-7, atol=0)


def test_pack_pose_meta_matches_data_layer_restatement(cuda):
    """pcnn_pack_pose_meta_fwd vs oracle.pack_pose_meta (minibatch.py:440-451, 474-492): row order / class / image columns
    exact, quaternions (Jacobi vs LAPACK eigh) and translations 1e-6, meta_data 1e-6 relative (cofactor inverse vs pinv)."""
    from scipy.spatial.transform import Rotation
    from posecnn_b200 import synth, train_ops
    rng = np.random.default_rng(9)
    B, I = 3, 5
    poses = np.zeros((B, I, 3, 4), np.float32)
    cls = -np.ones((B, I), np.int32)
    for b in range(B):
        n = [4, 0, 5][b]
        cls[b, :n] = rng.integers(1, 22, n)
        for j in range(n):
            poses[b, j, :, :3] = Rotation.from_quat(rng.normal(size=4)).as_matrix()
            poses[b, j, :, 3] = rng.uniform(-0.3, 1.2, 3)
    poses[0, 1, :, :3] = np.eye(3)                                          # identity rotation: degenerate eigenproblem
    poses[0, 2, :, :3] = Rotation.from_euler("z", 180, degrees=True).as_matrix()   # w = 0 boundary
    K = np.stack([synth.intrinsics(480, 640)] * B).astype(np.float32)
    for scale, flip in ((1.0, False), (0.5, True)):
        blob, nrows, meta = train_ops.pack_pose_meta(T(poses, cuda), T(cls, cuda), T(K, cuda), scale, flip)
        wb, wm = oracle.pack_pose_meta(poses, cls, K, scale, flip)
        n = int(nrows.item())
        assert n == wb.shape[0] == 9
        got = blob.cpu().numpy()
        assert not got[n:].any()
        np.testing.assert_array_equal(got[:n, :6], wb[:, :6])
        for a, b_ in zip(got[:n], wb):
            qa, qb = a[6:10], b_[6:10]
            if abs(qb[0]) < 1e-6:            # w = 0: the sign of the axis is arbitrary in both implementations
                qa = qa * np.sign(np.dot(qa, qb))
            np.testing.assert_allclose(qa, qb, atol=2e-6)
        np.testing.assert_allclose(got[:n, 10:], wb[:, 10:], atol=0)
        np.testing.assert_allclose(meta.cpu().numpy().reshape(B, 48), wm, rtol=1e-6, atol=1e-9)


def test_vertex_loss_from_lowres_equals_dense(cuda):
    """pcnn_vertex_loss_fused_lowres_fwd (vertex values formed on demand from the 1/8-resolution head tensor) == the fused loss on
    the dense vertex_pred produced by pcnn_up8_heads from the same tensor: the training step needs no dense vertex_pred."""
    from posecnn_b200 import synth, train_ops
    from posecnn_b200._lib import check, lib, ptr, stream
    B, H, W, C = 2, 96, 128, 22
    sc = synth.make_scene(batch=B, height=H, width=W, num_classes=C, seed=5, objects_per_image=4, min_pixels=100)
    g = torch.Generator().manual_seed(9)
    lowres = (torch.randn(B, H // 8, W // 8, 4 * C, generator=g) * 0.5).to(cuda)
    bs, bv = torch.zeros(C, device=cuda), (torch.randn(3 * C, generator=g) * 0.1).to(cuda)
    label = torch.empty((B, H, W), dtype=torch.int32, device=cuda)
    vertex = torch.empty((B, H, W, 3 * C), device=cuda)
    check(lib().pcnn_up8_heads(ptr(lowres), ptr(bs), ptr(bv), B, H // 8, W // 8, C, ptr(label), ptr(vertex), ptr(None), ptr(None), stream()))
    centers = np.zeros((B, C, 3), np.float32)
    for (b, cls, cx, cy, z) in sc["centers"]:
        centers[b, cls] = (cx, cy, z)
    lab, cen = T(sc["label"], cuda), T(centers, cuda)
    for sigma in (1.0, 2.0):
        l0, w0 = train_ops.vertex_loss_from_centers(vertex, lab, cen, 10.0, sigma, want_grad=False)
        out = torch.empty((2,), device=cuda)
        ws = train_ops._workspace(cuda)
        check(lib().pcnn_vertex_loss_fused_lowres_fwd(ptr(lowres), ptr(bv), ptr(lab), ptr(cen), B, H, W, C, 10.0, sigma, ptr(out), ptr(ws),
                                                      ws.numel(), stream()))
        assert float(w0.item()) == float(out[1].item()) > 0
        assert float(l0.item()) == float(out[0].item())
