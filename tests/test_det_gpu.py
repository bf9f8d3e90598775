"""The detection network (vgg16_det) on the device, stage by stage (DESIGN.md §16):

- RPN heads against an fp64 restatement on the same bf16 conv_rpn (structural 0.5 ties included);
- proposals: the decoded candidates within 2 ulp of bbox_transform_inv + clip_boxes on the device's own inputs, top-N and NMS
  exactly equal to the restatement on the device's own candidates (ties present), and the reference's outputs (det.npz);
- crop pool bit-exact against the CPU restatement (edge boxes, zero-width boxes, batch index > 0);
- the whole forward: heads against a torch fp32 chain on the device's own ROIs, batch invariance and CUDA-graph replay.
"""
import os

import numpy as np
import pytest
import torch

from tests import det_ref

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "det.npz"))
RATIOS = (0.5, 0.75, 1, 1.5, 2)
SCALES = {20: (4, 8, 16, 32), 30: (3, 4, 5, 6, 7, 8)}


def bf16_values(t):
    return t.float().cpu().numpy()


def rpn_inputs(cuda, B, h, w, A, seed, fg_shift=-0.5):
    """conv_rpn-like bf16 features (ReLU'd) and RPN weights whose biases push many logits below 0 (exact 0.5 ties)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, h, w, 512, generator=g)).to(torch.bfloat16)
    w_cls = torch.randn(1, 1, 512, 2 * A, generator=g) * (2.0 / 512) ** 0.5
    w_box = torch.randn(1, 1, 512, 4 * A, generator=g) * (0.02 / 512) ** 0.5
    b_cls = torch.randn(2 * A, generator=g) * 0.5 + fg_shift
    b_box = torch.randn(4 * A, generator=g) * 0.05 - 0.05
    return x.to(cuda), w_cls, b_cls, w_box, b_box


def run_rpn_heads(cuda, x, w_cls, b_cls, w_box, b_box, A):
    from posecnn_b200 import conv
    from posecnn_b200.rpn_layer.proposal_layer import rpn_heads
    w_tc = torch.cat([conv.hwio_to_tc(w_cls), conv.hwio_to_tc(w_box)]).to(cuda)
    bias = torch.cat([b_cls, b_box]).to(cuda)
    return rpn_heads(x, w_tc, bias, A)


@pytest.mark.parametrize("A", [20, 30])
def test_rpn_heads_against_fp64(cuda, A):
    x, w_cls, b_cls, w_box, b_box = rpn_inputs(cuda, 2, 30, 40, A, seed=A)
    prob, deltas = run_rpn_heads(cuda, x, w_cls, b_cls, w_box, b_box, A)
    wc = w_cls.to(torch.bfloat16).float().numpy()
    wb = w_box.to(torch.bfloat16).float().numpy()
    want_p, want_d = det_ref.rpn_heads(bf16_values(x), wc, b_cls.numpy(), wb, b_box.numpy())
    got_p, got_d = prob.cpu().numpy(), deltas.cpu().numpy()
    np.testing.assert_allclose(got_p, want_p, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got_d, want_d, rtol=1e-5, atol=1e-5 * float(np.abs(want_d).max()))
    assert (got_d >= 0).all()
    ties = got_p[..., A:] == 0.5
    assert int(ties.sum()) > 100, int(ties.sum())              # both logits of a pair ReLU'd to 0: probability exactly 0.5
    # where both fp64 logits are clearly <= 0 the device gives exactly 0.5; where one is clearly > 0 it does not (a logit within
    # fp32 accumulation error of 0 may fall either way)
    s64 = bf16_values(x).astype(np.float64) @ wc.reshape(512, -1).astype(np.float64) + b_cls.numpy().astype(np.float64)
    margin = 1e-4 * (np.abs(bf16_values(x)).astype(np.float64) @ np.abs(wc.reshape(512, -1)).astype(np.float64) + 1)
    clear_zero = (s64[..., :A] < -margin[..., :A]) & (s64[..., A:] < -margin[..., A:])
    clear_pos = (s64[..., :A] > margin[..., :A]) | (s64[..., A:] > margin[..., A:])
    assert ties[clear_zero].all() and not ties[clear_pos].any()


def test_rpn_heads_reject_foreign_operands(cuda):
    from posecnn_b200.rpn_layer.proposal_layer import rpn_heads
    A = 20
    x = torch.zeros((1, 2, 2, 512), dtype=torch.bfloat16, device=cuda)
    w = torch.zeros((6 * A, 512), dtype=torch.bfloat16, device=cuda)
    b = torch.zeros((6 * A,), dtype=torch.float32, device=cuda)
    with pytest.raises(TypeError):
        rpn_heads(x, w, b.double(), A)                         # a float64 bias
    with pytest.raises(RuntimeError):
        rpn_heads(x, w, b.cpu(), A)                            # a host bias
    with pytest.raises(RuntimeError):
        rpn_heads(x, w.cpu(), b, A)                            # host weights
    with pytest.raises(TypeError):
        rpn_heads(x, w.float(), b, A)


def check_image_proposals(b, prob, deltas, anchors, im_h, im_w, rois, scores, num, pre, post=300, pre_top_n=6000):
    """Image b's proposals against the restatement on the device's own inputs (decode) and own candidates (top-N order, NMS)."""
    A = prob.shape[-1] // 2
    s = prob[b, ..., A:].reshape(-1)
    order = det_ref.canonical_order(s)[:pre_top_n]
    K = order.size
    assert pre.shape[1] == K
    want_boxes, scale = det_ref.decode_clip(anchors, deltas[b].reshape(-1, 4), im_h, im_w, return_scale=True)
    np.testing.assert_array_equal(pre[b, :, 4], s[order])                     # the canonical order, ties by anchor index
    # expf and numpy's exp may differ in the last bit: within 2 ulp at the scale of the operands of x1 = ctr - w / 2
    assert (np.abs(pre[b, :, :4] - want_boxes[order]) <= 2 * np.spacing(scale[order])).all()
    keep = det_ref.nms_sorted(pre[b, :, :4], 0.7, post)
    n = int(num[b])
    assert n == keep.size
    rows = rois[b * post:(b + 1) * post]
    np.testing.assert_array_equal(rows[:n, 1:], pre[b, keep, :4])
    np.testing.assert_array_equal(scores[b * post:b * post + n, 0], pre[b, keep, 4])
    assert (rows[:, 0] == b).all() and (rows[n:, 1:] == 0).all() and (scores[b * post + n:(b + 1) * post] == 0).all()
    return n, K


@pytest.mark.parametrize("A,B,h,w", [(20, 1, 30, 40), (30, 4, 30, 40), (20, 4, 4, 5), (30, 1, 5, 7)])
def test_proposals_exact_with_ties(cuda, A, B, h, w):
    from posecnn_b200.rpn_layer.proposal_layer import proposals
    from posecnn_b200.rpn_layer.snippets import generate_anchors_pre
    x, w_cls, b_cls, w_box, b_box = rpn_inputs(cuda, B, h, w, A, seed=100 + A + B + h)
    prob, deltas = run_rpn_heads(cuda, x, w_cls, b_cls, w_box, b_box, A)
    anchors, _ = generate_anchors_pre(h, w, 16, SCALES[A], RATIOS)
    im_h, im_w = 16 * h, 16 * w
    rois, scores, num, pre = proposals(prob, deltas, torch.from_numpy(anchors).to(cuda), im_h, im_w, 6000, 300, 0.7,
                                       want_pre_boxes=True)
    p, d = prob.cpu().numpy(), deltas.cpu().numpy()
    assert np.unique(p[..., A:]).size < p[..., A:].size                      # exact ties among the candidates
    r, s, nn, pb = rois.cpu().numpy(), scores.cpu().numpy(), num.cpu().numpy(), pre.cpu().numpy()
    counts = [check_image_proposals(b, p, d, anchors, im_h, im_w, r, s, nn, pb) for b in range(B)]
    print("kept / candidates per image:", counts)
    if h * w * A < 6000:
        assert all(k == h * w * A for _, k in counts)
    if h * w <= 20:
        assert all(n < 300 for n, _ in counts)


@pytest.mark.parametrize("tag", ["lov", "linemod", "small", "few"])
def test_proposals_against_reference(cuda, tag):
    """The reference's proposal_layer (det.npz, tie-free inputs): its kept boxes, identified by their distinct scores among the
    device's sorted candidates, must be the device's keep list up to pairs whose fp64 IoU lies within 1e-6 of 0.7 (numpy's exp
    and the device's may differ in the last bit); every such difference is explained pair by pair (det_ref.explain_keep)."""
    from posecnn_b200.rpn_layer.proposal_layer import proposals
    fg = GOLD[f"{tag}_fg"]
    prob = np.concatenate([np.float32(1) - fg, fg], axis=-1)
    deltas = GOLD[f"{tag}_deltas"].astype(np.float32)
    im = GOLD[f"{tag}_im"]
    # two copies of the image: the second must give the same proposals, with batch index 1
    P = torch.from_numpy(np.concatenate([prob, prob])).to(cuda)
    D = torch.from_numpy(np.concatenate([deltas, deltas])).to(cuda)
    rois, scores, num, pre = proposals(P, D, torch.from_numpy(GOLD[f"{tag}_anchors"]).to(cuda), im[0], im[1], 6000, 300, 0.7,
                                       want_pre_boxes=True)
    r, s, n, pb = rois.cpu().numpy(), scores.cpu().numpy(), num.cpu().numpy(), pre.cpu().numpy()
    assert n[0] == n[1]
    np.testing.assert_array_equal(r[:300, 1:], r[300:, 1:])
    assert (r[:300, 0] == 0).all() and (r[300:, 0] == 1).all()
    pos = {float(v): k for k, v in enumerate(pb[0, :, 4])}                   # tie-free: a score names its candidate
    g_r, g_s = GOLD[f"{tag}_rois"], GOLD[f"{tag}_scores"]
    want = np.array([pos[float(v)] for v in g_s[:, 0]])
    # the reference's boxes are the device's candidates up to the last bit of exp() at image scale (2 ulp of 1024)
    assert np.abs(pb[0, want, :4] - g_r[:, 1:]).max() <= 2 * np.spacing(np.float32(1024))
    got = det_ref.nms_sorted(pb[0, :, :4], 0.7, 300)
    np.testing.assert_array_equal(r[:int(n[0]), 1:], pb[0, got, :4])
    flipped, amb = det_ref.explain_keep(pb[0, :, :4], 0.7, 300, want)
    print(f"{tag}: {len(amb)} candidate pairs within 1e-6 of IoU 0.7, {len(flipped)} decided the other way by the reference")


def load_ref_nms():
    import ctypes
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_nms.so")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/libref_nms.so was not built (needs a checkout of the reference: oracle/ref_nms.mk)")
    lib = ctypes.CDLL(path)
    lib.ref_gpu_nms.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int]
    lib.ref_gpu_nms.restype = ctypes.c_int
    return lib


def ref_gpu_nms(lib, boxes5, thresh, device_id):
    import ctypes
    b = np.ascontiguousarray(boxes5, dtype=np.float32)
    keep = np.zeros(b.shape[0], dtype=np.int32)
    num = ctypes.c_int(0)
    rc = lib.ref_gpu_nms(keep.ctypes.data, ctypes.addressof(num), b.ctypes.data, b.shape[0], thresh, device_id)
    assert rc == 0, rc
    return keep[:num.value].astype(np.int64)


@pytest.mark.parametrize("A,B,h,w", [(20, 2, 30, 40), (30, 2, 30, 40), (20, 1, 4, 5)])
def test_nms_against_reference_kernel(cuda, A, B, h, w):
    """The device's keep list against the reference's own nms_kernel.cu (oracle/ref_nms.cu, FMA contraction as nvcc compiles
    it) on the device's sorted candidates, ties present: equal up to pairs whose fp64 IoU lies within 1e-6 of 0.7, which are
    counted and reported."""
    from posecnn_b200.rpn_layer.proposal_layer import proposals
    from posecnn_b200.rpn_layer.snippets import generate_anchors_pre
    lib = load_ref_nms()
    x, w_cls, b_cls, w_box, b_box = rpn_inputs(cuda, B, h, w, A, seed=300 + A + B + h)
    prob, deltas = run_rpn_heads(cuda, x, w_cls, b_cls, w_box, b_box, A)
    anchors, _ = generate_anchors_pre(h, w, 16, SCALES[A], RATIOS)
    rois, scores, num, pre = proposals(prob, deltas, torch.from_numpy(anchors).to(cuda), 16 * h, 16 * w, 6000, 300, 0.7,
                                       want_pre_boxes=True)
    torch.cuda.synchronize()
    r, nn, pb = rois.cpu().numpy(), num.cpu().numpy(), pre.cpu().numpy()
    for b in range(B):
        mine = det_ref.nms_sorted(pb[b, :, :4], 0.7, 300)
        np.testing.assert_array_equal(r[b * 300:b * 300 + int(nn[b]), 1:], pb[b, mine, :4])    # the device's own keep list
        theirs = ref_gpu_nms(lib, pb[b], 0.7, cuda.index or 0)[:300]          # proposal_layer.py: keep[:post_nms_topN]
        flipped, amb = det_ref.explain_keep(pb[b, :, :4], 0.7, 300, theirs)
        print(f"image {b}: kept {mine.size} / {theirs.size}; {len(amb)} candidate pairs within 1e-6 of IoU 0.7, "
              f"{len(flipped)} decided differently by the reference kernel")


def test_crop_pool_bit_exact(cuda):
    from posecnn_b200 import pose_head
    g = torch.Generator().manual_seed(5)
    B, H, W, C = 3, 30, 40, 512
    feat = (torch.randn(B, H, W, C, generator=g) * 3).to(torch.bfloat16)
    im_w, im_h = 640.0, 480.0
    rows = []
    rng = np.random.default_rng(5)
    for i in range(24):                                        # random boxes, every image
        x1, y1 = rng.uniform(0, im_w - 1), rng.uniform(0, im_h - 1)
        rows.append([i % B, x1, y1, rng.uniform(x1, im_w - 1), rng.uniform(y1, im_h - 1)])
    rows += [[1, 300.0, 200.0, im_w - 1, im_h - 1], [2, 0.0, 0.0, im_w - 1, im_h - 1],    # right / bottom edges: extrapolation zeros
             [2, 600.5, 100.0, im_w - 1, 110.0], [0, 10.0, 470.0, 50.0, im_h - 1],
             [1, 123.0, 40.0, 123.0, 300.0], [2, 50.0, 77.0, 400.0, 77.0], [0, 320.0, 240.0, 320.0, 240.0],   # zero width / height
             [1, 0.0, 0.0, 0.0, 0.0], [2, 0.0, 0.0, 0.0, 0.0]]                                            # capacity rows
    rois = np.asarray(rows, dtype=np.float32)
    got = pose_head.crop_pool(feat.to(cuda), torch.from_numpy(rois).to(cuda), 16.0).cpu().numpy()
    want = det_ref.crop_pool(bf16_values(feat), rois, 16.0)
    assert got.shape == (rois.shape[0], 7 * 7 * C)
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    edge = want.reshape(-1, 7, 7, C)[24]
    assert (edge[-1] == 0).any() or (edge[:, -1] == 0).any()


def images(B, H, W, seed):
    from posecnn_b200 import synth
    rgb, _ = synth.make_images(B, H, W, seed=seed)
    return torch.from_numpy(np.ascontiguousarray(rgb))


def rel_l2(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("C,A", [(22, 20), (2, 30)])
def test_forward_heads_against_fp32(cuda, C, A):
    from posecnn_b200.networks import vgg16_det
    net = vgg16_det(num_classes=C, anchor_scales=SCALES[A], device=cuda).init_random(seed=C, bias_std=0.05)
    data = images(2, 480, 640, seed=C).to(cuda)
    L = net.forward(data, sync_rois=False)
    N = 300
    assert L["rpn_cls_prob"].shape == (2, 30, 40, 2 * A) and L["rpn_bbox_pred"].shape == (2, 30, 40, 4 * A)
    assert L["rois"].shape == (2 * N, 5) and L["rpn_scores"].shape == (2 * N, 1) and L["num_rois"].dtype == torch.int32
    assert L["cls_prob"].shape == (2 * N, C) and L["bbox_pred"].shape == (2 * N, 4 * C) and L["poses_tanh"].shape == (2 * N, 4 * C)
    rois = L["rois"].cpu().numpy()
    num = L["num_rois"].cpu().numpy()
    assert (num >= 1).all() and (num <= N).all()
    assert (rois[:N, 0] == 0).all() and (rois[N:, 0] == 1).all()
    x = torch.from_numpy(det_ref.crop_pool(bf16_values(L["conv5_3"]), rois, 16.0)).to(cuda).float()
    P = net.params
    h = torch.relu(x @ P["fc6/weights"] + P["fc6/biases"])
    h = torch.relu(h @ P["fc7/weights"] + P["fc7/biases"])
    cls_prob = torch.softmax(torch.relu(h @ P["cls_score/weights"] + P["cls_score/biases"]), dim=1)
    bbox = h @ P["bbox_pred/weights"] + P["bbox_pred/biases"]
    poses = torch.tanh(h @ P["poses_pred_unnormalized/weights"] + P["poses_pred_unnormalized/biases"])
    # fp16 weights and fp16 fc6 / fc7 activations against fp32 throughout
    assert rel_l2(L["cls_prob"], cls_prob) < 1e-2
    assert rel_l2(L["bbox_pred"], bbox) < 1e-2
    assert rel_l2(L["poses_tanh"], poses) < 1e-2
    torch.testing.assert_close(L["cls_prob"].sum(1), torch.ones(2 * N, device=cuda), rtol=0, atol=1e-5)
    # sync_rois: the rows each image keeps, in order
    S = net.forward(data, sync_rois=True)
    idx = np.concatenate([np.arange(b * N, b * N + num[b]) for b in range(2)])
    for k in ("rois", "rpn_scores", "cls_prob", "bbox_pred", "poses_tanh"):
        assert torch.equal(S[k], L[k][torch.from_numpy(idx).to(cuda)]), k


def test_batch_invariance(cuda):
    from posecnn_b200.networks import vgg16_det
    net = vgg16_det(num_classes=22, device=cuda).init_random(seed=7, bias_std=0.05)
    data = images(4, 480, 640, seed=7).to(cuda)
    L = {k: v.clone() for k, v in net.forward(data, sync_rois=False).items()}
    N = 300
    for b in range(4):
        one = net.forward(data[b:b + 1].contiguous(), sync_rois=False)
        for k in ("rpn_cls_prob", "rpn_bbox_pred", "num_rois"):
            assert torch.equal(one[k], L[k][b:b + 1]), (b, k)
        for k in ("rpn_scores", "cls_prob", "bbox_pred", "poses_tanh"):
            assert torch.equal(one[k], L[k][b * N:(b + 1) * N]), (b, k)
        assert torch.equal(one["rois"][:, 1:], L["rois"][b * N:(b + 1) * N, 1:]), b
        assert (L["rois"][b * N:(b + 1) * N, 0] == b).all()


def test_graph_replay_equals_eager(cuda):
    from posecnn_b200.networks.vgg16_det import GraphedForward, vgg16_det
    net = vgg16_det(num_classes=2, anchor_scales=SCALES[30], device=cuda).init_random(seed=3, bias_std=0.05)
    first = images(2, 480, 640, seed=11).to(cuda)
    second = images(2, 480, 640, seed=12).to(cuda)
    graphed = GraphedForward(net, first)
    got = {k: v.clone() for k, v in graphed(second).items()}
    torch.cuda.synchronize()
    want = net.forward(second, sync_rois=False)
    for k in ("rpn_cls_prob", "rois", "rpn_scores", "num_rois", "cls_prob", "bbox_pred", "poses_tanh"):
        assert torch.equal(got[k], want[k]), k
