"""GPU parity of the training-side target generation and the training step's losses (SURVEY.md §8(f) rank 3) against the
reference's own _generate_vertex_targets output (tests/golden/vertex_targets.npz) and the numpy restatements of the TF loss graphs."""
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


def _scene_centres(label, C, rng, jitter):
    """centers [B,C,3] of every labelled class of each image: its pixels' mean (+ N(0, jitter) per axis) and a depth in [0.5, 1.5)."""
    centers = np.zeros((label.shape[0], C, 3), np.float32)
    for b in range(label.shape[0]):
        for c in np.unique(label[b]):
            if c > 0:
                ys, xs = np.where(label[b] == c)
                centers[b, c] = (xs.mean() + jitter * rng.normal(), ys.mean() + jitter * rng.normal(), rng.uniform(0.5, 1.5))
    return centers


def test_step_losses_against_oracle(cuda):
    """configs[4] shape in miniature (a GPU's share of the batch): Trainer.forward -> Hough in train mode (9 jittered rows per ROI,
    quaternion targets from the gt poses) -> RoiPool -> pose head, and the step's three losses, each against the oracle on the
    step's own intermediate tensors: cls_out on the float64 log-softmax of A["score"], vtx_out on the dense vertex_pred of the
    same heads (Trainer.dense_vertex_pred) and the oracle's targets, loss_pose_raw by Averagedistance on A's pose rows."""
    from posecnn_b200 import synth
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.train import Trainer
    from tests.train_ref import synthetic_pose_targets
    C, B, H, W = 6, 2, 64, 96
    net = vgg16_convs(num_classes=C, device=cuda, is_train=True, fold_vertex_head=False).init_random(seed=0, bias_std=0.05)
    tr = Trainer(net)
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
    points = T(synth.make_model_points(C, 200, seed=2), cuda)
    symmetry = torch.zeros((C,), device=cuda); symmetry[2] = 1.0
    # the network's own labels (they do not depend on the gt inputs) -> gt labels with 10 % ignore and 30 % disagreeing pixels
    zeros = torch.zeros((B, H, W), dtype=torch.int32, device=cuda), torch.zeros((B, C, 3), device=cuda)
    label = to_np(tr.forward(data, *zeros, meta, ext, T(gt, cuda), points, symmetry)["label_2d"])
    u = rng.random(label.shape)
    gt_label = np.where(u < 0.1, -1, np.where(u < 0.4, rng.integers(0, C, label.shape), label)).astype(np.int32)
    centers = _scene_centres(label, C, rng, 0.0)
    A = tr.forward(data, T(gt_label, cuda), T(centers, cuda), meta, ext, T(gt, cuda), points, symmetry)
    # classification: log-softmax of the step's own scores, Hardlabel selection
    score = to_np(A["score"]).astype(np.float64)
    logp = score - np.log(np.exp(score - score.max(3, keepdims=True)).sum(3, keepdims=True)) - score.max(3, keepdims=True)
    want_cls, mask = oracle.loss_cross_entropy_hard(logp, to_np(A["prob_normalized"]), gt_label, net.threshold_label)
    assert float(A["cls_out"][1].item()) == mask.sum()
    assert want_cls > 1e-3 and abs(float(A["cls_out"][0].item()) - want_cls) <= 2e-5 * abs(want_cls)
    vt, vw = oracle.generate_vertex_targets(gt_label, centers, tr.w_inside)
    want_v, _ = oracle.smooth_l1_loss_vertex(to_np(tr.dense_vertex_pred(A)), vt, vw, 1.0)
    assert float(A["vtx_out"][1].item()) == float(vw.astype(np.float64).sum()) > 0
    assert abs(float(A["vtx_out"][0].item()) - want_v) <= 1e-5 * abs(want_v)
    # pose: rows come in groups of 9 per ROI in train mode; weights select the gt class quaternion
    assert A["rois"].shape[0] % 9 == 0 and A["poses_weight"].shape == A["poses_tanh"].shape
    # on Hough's targets, then (their weights are all 0 on this scene) on quaternion targets of the rows' own classes, which
    # train_ref.synthetic_pose_targets runs through the step's Averagedistance
    for _ in range(2):
        pt, pw, ptg = to_np(A["poses_tanh"]), to_np(A["poses_weight"]), to_np(A["poses_target"])
        mul = pt * pw
        pred = mul / np.sqrt(np.maximum((mul ** 2).sum(1, keepdims=True), 1e-12))
        want_p, _ = oracle.average_distance_loss(pred.astype(np.float32), ptg, pw, to_np(points), to_np(symmetry), tr.margin)
        assert abs(float(A["loss_pose_raw"].item()) - float(want_p[0])) <= 1e-4 * max(abs(float(want_p[0])), 1e-6)
        synthetic_pose_targets(A, points, symmetry, tr.margin)
    assert pw.any() and float(want_p[0]) > 0


@pytest.mark.parametrize("sigma", [1.0, 2.5])
def test_loss_vertex_full_frame(cuda, sigma):
    """train_ops.loss_vertex (the step's loss_vertex: vertex values formed from the 1/8-resolution head tensor, targets never
    materialised) at 2 x 480 x 640, C = 22, with one labelled class not listed, against
    oracle.smooth_l1_loss_vertex (fp32 terms, float64 sum) on the dense vertex_pred that pcnn_up8_heads writes from the same tensor
    and the oracle's targets: sum of weights exact, two launches bit-identical, and the loss within 1e-6 relative.  That bound is the
    one the fused kernel was held to against smooth L1 on the materialised blobs: the vertex values are bit-identical to the dense
    tensor's, the targets are the oracle's to 1 ulp of log z, each term is the same fp32 expression, and the float64 sums differ
    only in order, so the quotient's fp32 rounding (2^-24 relative) dominates."""
    from posecnn_b200 import heads, synth, train_ops
    B, H, W, C = 2, 480, 640, 22
    sc = synth.make_scene(batch=B, height=H, width=W, num_classes=C, seed=77)
    label = sc["label"]
    centers = _scene_centres(label, C, np.random.default_rng(2), 1.0)
    c0 = int(np.unique(label[0])[1])
    centers[0, c0, 2] = 0.0                                            # one labelled class not listed
    g = torch.Generator().manual_seed(9)
    lowres = (torch.randn(B, H // 8, W // 8, 4 * C, generator=g) * 0.5).to(cuda)
    bs, bv = torch.zeros(C, device=cuda), (torch.randn(3 * C, generator=g) * 0.1).to(cuda)
    vertex = heads.up8_heads(lowres, bs, bv, vertex=True)[1]
    vp = to_np(vertex)
    vt, vw = oracle.generate_vertex_targets(label, centers, 10.0)
    assert (label[0] == c0).any() and not vw[0, ..., 3 * c0:3 * c0 + 3].any()
    lab, cen = T(label, cuda), T(centers, cuda)
    out = train_ops.loss_vertex(lowres, bv, lab, cen, 10.0, sigma)
    again = train_ops.loss_vertex(lowres, bv, lab, cen, 10.0, sigma)
    want, _ = oracle.smooth_l1_loss_vertex(vp, vt, vw, sigma)
    d = np.abs(vw * (vp - vt))[vw > 0]
    print(f"sigma {sigma}: loss {out[0].item():.7f} oracle {want:.7f}; {(d < 1 / sigma ** 2).mean():.2f} of the weighted terms quadratic")
    assert (d < 1 / sigma ** 2).any() and (d >= 1 / sigma ** 2).any()
    assert float(out[1].item()) == float(vw.astype(np.float64).sum()) > 0
    assert abs(float(out[0].item()) - want) <= 1e-6 * abs(want)
    assert torch.equal(out, again)


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
