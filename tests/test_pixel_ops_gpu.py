"""GPU parity of RoiPool, Hardlabel, Averagedistance (C ABI) vs the CPU oracle (Backproject / Project: test_project_exact_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import oracle
from posecnn_b200 import synth
from tests.util import to_np

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.mark.parametrize("channels,pool_channel", [(512, 0), (30, 0), (22, 1)])
def test_roi_pool_fwd_bwd(cuda, channels, pool_channel):
    from posecnn_b200.roi_pooling_layer import roi_pooling_op as op
    rng = np.random.default_rng(0)
    B, h, w = 3, 30, 40
    data = rng.standard_normal((B, h, w, channels)).astype(np.float32)
    rois = synth.make_rois(17, B, num_classes=min(22, channels), seed=2)
    rois[3, 2:6] = [700, 500, 710, 505]          # outside the image -> empty bins
    rois[4, 2:6] = [100, 100, 90, 80]            # malformed -> forced 1x1
    top_w, arg_w = oracle.roi_pool(data, rois, 7, 7, 1.0 / 16.0, pool_channel)
    top, arg = op.roi_pool(T(data, cuda), T(rois, cuda), 7, 7, 1.0 / 16.0, pool_channel)
    np.testing.assert_array_equal(to_np(arg), arg_w)          # index work: bit exact
    np.testing.assert_array_equal(to_np(top), top_w)
    g = rng.standard_normal(top_w.shape).astype(np.float32)
    gin_w = oracle.roi_pool_grad(data, rois, arg_w, g, 7, 7, 1.0 / 16.0, pool_channel)
    gin = op.roi_pool_grad(T(data, cuda), T(rois, cuda), arg, T(g, cuda), 7, 7, 1.0 / 16.0, pool_channel)
    np.testing.assert_allclose(to_np(gin), gin_w, rtol=1e-5, atol=1e-6)   # float atomics: summation order only


def test_roi_pool_autograd(cuda):
    from posecnn_b200.roi_pooling_layer import roi_pooling_op_grad as opg
    rng = np.random.default_rng(1)
    data = T(rng.standard_normal((2, 12, 16, 8)).astype(np.float32), cuda).requires_grad_()
    rois = T(synth.make_rois(5, 2, height=96, width=128, seed=3), cuda)
    top, arg = opg.roi_pool(data, rois, 7, 7, 1.0 / 8.0, 0)
    top.sum().backward()
    m = to_np(arg) >= 0
    assert abs(float(data.grad.sum()) - m.sum()) < 1e-3


@pytest.mark.parametrize("C", [22, 5])
def test_hard_label(cuda, C):
    from posecnn_b200.hard_label_layer import hard_label_op as op
    rng = np.random.default_rng(2)
    prob = rng.random((2, 37, 53, C)).astype(np.float32)
    gt = rng.integers(-1, C, (2, 37, 53)).astype(np.int32)
    for thr in (1.0, 0.5, 0.0):
        out = op.hard_label(T(prob, cuda), T(gt, cuda), thr)
        np.testing.assert_array_equal(to_np(out), oracle.hard_label(prob, gt, thr))
    gp, gg = op.hard_label_grad(T(prob, cuda), T(gt, cuda), out)
    assert gp.shape == (2, 37, 53, C) and gg.shape == (2, 37, 53) and not gp.any() and not gg.any()


@pytest.mark.parametrize("P,N", [(2620, 18), (300, 5)])
def test_average_distance(cuda, P, N):
    from posecnn_b200.average_distance_loss import average_distance_loss_op as op
    from posecnn_b200.average_distance_loss import average_distance_loss_op_grad as opg
    pts = synth.make_model_points(22, P)
    pred, targ, wt = synth.make_pose_batch(N, 22, seed=9)
    # make sure a symmetric class (16 or 21, lib/datasets/lov.py:38) is present
    pred[0] = 0; targ[0] = 0; wt[0] = 0
    q = np.array([0.8, 0.2, -0.4, 0.4], np.float32); p = q + np.array([0.1, -0.05, 0.02, 0.07], np.float32)
    targ[0, 64:68] = q / np.linalg.norm(q); pred[0, 64:68] = p / np.linalg.norm(p); wt[0, 64:68] = 1
    sym = synth.LOV_SYMMETRY
    loss_w, diff_w = oracle.average_distance_loss(pred, targ, wt, pts, sym, 0.01)
    a = [T(x, cuda) for x in (pred, targ, wt, pts, sym)]
    loss, diff = op.average_distance_loss(*a, 0.01)
    np.testing.assert_allclose(to_np(loss), loss_w, rtol=1e-4)                       # stated tolerance: rel 1e-4
    np.testing.assert_allclose(to_np(diff), diff_w, rtol=1e-3, atol=1e-4 * np.abs(diff_w).max())
    loss2, _ = op.average_distance_loss(*a, 0.01)
    assert float(loss2) == float(loss)                                               # deterministic reduction
    pr = a[0].clone().requires_grad_()
    l, _ = opg.average_distance_loss(pr, *a[1:], 0.01)
    (3.0 * l).sum().backward()
    np.testing.assert_allclose(to_np(pr.grad), 3.0 * to_np(diff), rtol=1e-6)         # AveragedistanceGrad = upstream * diff


@pytest.mark.parametrize("channels", [512, 128, 72])
def test_roi_pool_bf16_features_with_ties(cuda, channels):
    """bf16 feature maps (what the tensor-core trunk hands over): channels % 64 == 0 takes the sliced kernel whose
    shuffle merge must reproduce the raster-order first-maximum rule.  Small-integer features force many ties."""
    from posecnn_b200.roi_pooling_layer import roi_pooling_op as op
    rng = np.random.default_rng(7)
    B, h, w = 2, 60, 80
    data = rng.integers(-2, 3, size=(B, h, w, channels)).astype(np.float32)      # exactly representable in bf16
    rois = synth.make_rois(23, B, num_classes=22, seed=9)
    rois[0, 2:6] = [0, 0, 639, 479]              # whole image: large bins
    rois[1, 2:6] = [16, 16, 23, 23]              # one feature cell
    rois[2, 2:6] = [900, 900, 910, 910]          # outside
    top_w, arg_w = oracle.roi_pool(data, rois, 7, 7, 1.0 / 8.0, 0)
    top, arg = op.roi_pool(T(data, cuda).to(torch.bfloat16), T(rois, cuda), 7, 7, 1.0 / 8.0, 0)
    np.testing.assert_array_equal(to_np(arg), arg_w)
    np.testing.assert_array_equal(to_np(top), top_w)
