"""Parity at the BASELINE size: the whole network at 480x640, C = 22 (batch 2) against the fp32 restatement of the
reference graph (oracle/ref_network.py), the Hough rows of the pipeline against the C oracle on the pipeline's own
maps, the calibration helper of the benchmark harness, and the depth blob fused into conv1_1_p.
Tolerances: SURVEY.md §8(c) — trunk rel-L2 <= 2e-2 (BF16 operands), labels compared under a logit-margin mask,
integer fields exact, boxes / poses 1e-4, tanh quaternions abs 1e-3 against the fp32 head on the same features."""
import numpy as np
import pytest
import torch

from oracle import oracle
from posecnn_b200 import synth
from tests import ref_network as R
from tests.util import to_np

pytestmark = pytest.mark.gpu
MEANS = (102.9801, 115.9465, 122.7717)


def rel_l2(a, b):
    return ((a - b).pow(2).sum() / b.pow(2).sum().clamp(min=1e-30)).sqrt().item()


@pytest.fixture(scope="module")
def full(cuda):
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    B, H, W, C = 2, 480, 640, 22
    net = vgg16_convs(num_classes=C, device=cuda).init_random(seed=0)
    rgb, _ = synth.make_images(B, H, W, seed=3)
    data = torch.from_numpy(rgb).to(cuda)
    meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)).to(cuda)
    ext = torch.from_numpy(synth.extents_for(C)).to(cuda)
    shift = net.calibrate_background(data, meta, ext, 0.75)
    out = dict(net.forward(data, meta, ext, want_prob=True, want_score=True))
    torch.cuda.synchronize()
    return net, data, meta, ext, out, shift


def test_calibrate_background_hits_the_requested_fill(full):
    net, data, meta, ext, out, shift = full
    bg = (out["label_2d"] == 0).float().mean().item()
    assert abs(bg - 0.75) < 0.02, bg
    assert shift > 0          # the un-calibrated random-init net labels (almost) everything foreground


def test_trunk_and_heads_480x640(full):
    """conv4_3 / conv5_3 rel-L2 vs fp32 cuDNN (TF32 off), vertex_pred rel-L2, label flip rate under a margin mask."""
    net, data, meta, ext, out, _ = full
    x = (data.float() - torch.tensor(MEANS, device=data.device)).permute(0, 3, 1, 2)
    with torch.no_grad():
        feats = R.trunk(net.params, x)
        for name in ("conv4_3", "conv5_3"):
            e = rel_l2(out[name].float().permute(0, 3, 1, 2), feats[name])
            assert e < 2e-2, (name, e)
        score, label, prob, vertex = R.heads(net.params, feats["conv4_3"], feats["conv5_3"], 22)
    assert rel_l2(out["vertex_pred"].permute(0, 3, 1, 2), vertex) < 2e-2
    top2 = torch.topk(score, 2, dim=1).values
    margin = (top2[:, 0] - top2[:, 1]) / top2[:, 0].abs().clamp(min=1e-6)
    decided = margin > 0.05                                   # fp32 logit margin > 5 %: a bf16 trunk must not flip these
    frac = decided.float().mean().item()
    flips = (out["label_2d"][decided] != label[decided]).float().mean().item()
    flips_all = (out["label_2d"] != label).float().mean().item()
    print(f"480x640: {frac:.3f} of pixels decided by > 5 %; flip rate there {flips:.2e}, over all pixels {flips_all:.2e}")
    assert frac > 0.3 and flips < 1e-3
    assert torch.allclose(out["prob_normalized"].sum(3), torch.ones_like(out["prob_normalized"][..., 0]), atol=1e-5)


def test_hough_rows_vs_oracle_on_network_maps(full):
    """Houghvotinggpu inside the pipeline == the C oracle on the pipeline's own label / vertex maps (image 0 alone: the
    oracle's per-cell loops take ~10 s per frame on these noise-like maps), and == the batch rows of that image."""
    net, data, meta, ext, out, _ = full
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    lab, ver = out["label_2d"][:1].contiguous(), out["vertex_pred"][:1].contiguous()
    want = oracle.hough_voting_gpu(to_np(lab), to_np(ver), to_np(ext), to_np(meta[:1]), None, 0, -1.0, 0.02, 10)
    got = [to_np(t) for t in op.hough_voting_gpu(lab, ver, ext, meta[:1], None, 0, -1.0, 0.02, 10)]
    assert got[0].shape == want[0].shape and got[0].shape[0] >= 2
    np.testing.assert_array_equal(got[0][:, [0, 1, 6]], want[0][:, [0, 1, 6]])
    np.testing.assert_allclose(got[0][:, 2:6], want[0][:, 2:6], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-4, atol=1e-4)
    # the batch-of-2 rows of image 0 are the first 128 // 2 classes of the single-image result
    rows = to_np(out["rois"])
    r0 = rows[rows[:, 0] == 0]
    k = r0.shape[0]
    assert k == min(64, got[0].shape[0])
    np.testing.assert_array_equal(r0, got[0][:k])


def test_pose_head_480x640_against_fp32_head(full):
    """RoiPool-pair + fc6-fc8 (+ tanh) on the tensor cores vs the fp32 torch head on the SAME conv features and ROIs.
    The head runs on FP16 operands (11-bit mantissa; BF16 left 4.8e-3 rel-L2 on the fc8 pre-activations and 2.8e-3 abs on the
    quaternions, measured): stated tolerance rel-L2 <= 1.5e-3 on the fc6 / fc7 activations and the fc8 pre-activations;
    tanh quaternions abs 1e-3 (SURVEY §8(c)) with the pre-activations scaled to O(0.2)
    (a Kaiming-initialised fc8 emits pre-activations of several hundred, where tanh is +-1 and the comparison is void)."""
    from posecnn_b200 import pose_head
    net, data, meta, ext, out, _ = full
    rois = to_np(out["rois"])
    p5, _ = oracle.roi_pool(to_np(out["conv5_3"].float()), rois, 7, 7, 1.0 / 16.0)
    p4, _ = oracle.roi_pool(to_np(out["conv4_3"].float()), rois, 7, 7, 1.0 / 8.0)
    x0 = torch.from_numpy(p5 + p4).reshape(rois.shape[0], -1).to(data.device)
    n = rois.shape[0]
    assert torch.equal(out["pool_score"][:n], x0.to(torch.float16))            # fused pooling == oracle RoiPool x2 + add, rounded once
    P, T = net.params, net._tc
    h6 = torch.relu(x0 @ P["fc6/weights"] + P["fc6/biases"])
    h7 = torch.relu(h6 @ P["fc7/weights"] + P["fc7/biases"])
    pre = h7 @ P["fc8/weights"] + P["fc8/biases"]
    assert rel_l2(out["fc6"][:n, :4096].float(), h6) < 1.5e-3
    assert rel_l2(out["fc7"][:n, :4096].float(), h7) < 1.5e-3
    got_pre = pose_head.fc(out["fc7"][:n].contiguous(), T["fc8/weights"], P["fc8/biases"], "none", torch.float32)
    e_pre = rel_l2(got_pre, pre)
    scale = 0.2 / pre.std().item()
    w8 = pose_head.fc_weights_to_tc(P["fc8/weights"] * scale)
    got = pose_head.fc(out["fc7"][:n].contiguous(), w8, P["fc8/biases"] * scale, "tanh", torch.float32)
    err = (got - torch.tanh(pre * scale)).abs().max().item()
    print(f"pose head: fc8 pre-activation rel-L2 {e_pre:.2e}; tanh abs err at O(0.2) pre-activations {err:.2e}")
    assert e_pre < 1.5e-3 and err < 1e-3, (e_pre, err)


def _depth_blob_case(cuda, B, H, W):
    from posecnn_b200 import conv
    from posecnn_b200.utils import blob
    g = np.random.default_rng(5)
    depth = g.uniform(-100.0, 2600.0, (B, H, W)).astype(np.float32)      # mm; values below 0 and above 2000 exercise the clip
    depth[0, :3] = 0.0
    w = torch.randn((3, 3, 3, 64), generator=torch.Generator().manual_seed(1)) * 0.1
    bias = torch.randn(64, generator=torch.Generator().manual_seed(2)) * 0.1
    w_tc = conv.conv1_1_weights_to_tc(w.to(cuda))
    host_blob = torch.from_numpy(blob.depth_blob([d for d in depth])).to(cuda)
    want = conv.conv1_fused(host_blob, w_tc, bias.to(cuda), None, True)
    got = conv.conv1_depth_fused(torch.from_numpy(depth).to(cuda), w_tc, bias.to(cuda), MEANS, True)
    assert torch.equal(got, want)


def test_depth_blob_fused_into_conv1(cuda):
    """f2: conv1_1_p on the RAW depth image (blob clip(d / 2000, 0, 1) * 255 x3 - PIXEL_MEANS formed in the loader,
    lib/fcn/test.py:70-76) == the same kernel fed the host-side blob of posecnn_b200/utils/blob.py: bit-identical."""
    _depth_blob_case(cuda, 2, 48, 80)


def test_depth_blob_fused_into_conv1_480x640(cuda):
    """The same at 480 x 640: every CTA runs 36 tiles, so all four builder groups and both consumer warpgroups take part."""
    _depth_blob_case(cuda, 2, 480, 640)


def test_rgbd_network_with_raw_depth_input(cuda):
    """RGBD network fed the raw depth image (depth=) == fed the host-side depth blob (data_p=)."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.utils import blob
    net = vgg16_convs(input_format="RGBD", num_classes=4, device=cuda).init_random(seed=1, bias_std=0.05)
    rgb, depth = synth.make_images(2, 48, 64, seed=5)
    dmm = (depth * 1000.0).astype(np.float32)
    data = torch.from_numpy(rgb).to(cuda)
    meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(48, 64))] * 2)).to(cuda)
    ext = torch.from_numpy(synth.extents_for(4)).to(cuda)
    a = dict(net.forward(data, meta, ext, data_p=torch.from_numpy(blob.depth_blob([d for d in dmm])).to(cuda), sync_rois=False))
    b = dict(net.forward(data, meta, ext, depth=torch.from_numpy(dmm).to(cuda), sync_rois=False))
    for k in ("label_2d", "vertex_pred", "rois_capacity", "poses_tanh"):
        assert torch.equal(a[k], b[k]), k
