"""Image scale on the GPU (csrc/rescale.cu, posecnn_b200/rescale.py) and the object-coordinate path at the resolution the LINEMOD
*_3d.yml models run (SCALES_BASE 1.5: 480 x 640 frames become 720 x 960 images): every resize mode bit for bit against
tests/rescale_ref.py, the training inputs against the data layer's order of operations, the convolutions at the 720 x 960 layer
shapes exactly, the C = 2 network forward and training step against fp32 references, a planted scene through the test-time flow,
and conv1 above 2^31 activation elements.  Every measured error is printed."""
import numpy as np
import pytest
import torch

from posecnn_b200 import synth
from tests import rescale_ref as ref
from tests.train_ref import rel_l2

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
S = 1.5
CASES = [(480, 640, S), (37, 53, S), (37, 53, 1.25), (480, 640, 1.0)]


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def u16(a, dev):
    return T(np.ascontiguousarray(a, np.uint16).view(np.int16), dev).view(torch.uint16)


def same_bits(got, want):
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (g.shape, w.shape, g.dtype, w.dtype)
    bad = int((g.view(np.uint8).reshape(g.shape + (-1,)) != w.view(np.uint8).reshape(w.shape + (-1,))).any(-1).sum())
    assert bad == 0, f"{bad} of {g.size} values differ"


def ints(t):
    """uint16 tensors compared through their int16 view (few torch ops take uint16)."""
    return t.view(torch.int16) if t.dtype == torch.uint16 else t


def _inputs(B, H, W, seed):
    g = np.random.default_rng(seed)
    depth = g.integers(300, 4000, (B, H, W)).astype(np.uint16)
    depth[:, H // 3: H // 2, W // 4: W // 2] = 0
    depth[0, :4, :] = 65535
    return dict(frames=g.integers(0, 256, (B, H, W, 3), dtype=np.uint8),
                x3=((g.random((B, H, W, 3)) - 0.5) * 250).astype(np.float32),
                x1=((g.random((B, H, W)) - 0.5) * 2).astype(np.float32),
                depth=depth, label=g.integers(-1, 9, (B, H, W)).astype(np.int32))


def _run_all(rescale, I, s, dev):
    return dict(color=rescale.color_blob(T(I["frames"], dev), s), x3=rescale.resize_linear(T(I["x3"], dev), s),
                x1=rescale.resize_linear(T(I["x1"], dev), s), d16=rescale.resize_depth(u16(I["depth"], dev), s),
                d32=rescale.resize_depth(T(I["depth"].astype(np.float32), dev), s), label=rescale.resize_nearest(T(I["label"], dev), s))


@pytest.mark.parametrize("H,W,s", CASES, ids=[f"{h}x{w}@{s}" for h, w, s in CASES])
def test_every_mode_equals_restatement(cuda, H, W, s):
    """Batch 3; each image of the batch resized alone equals its row of the batch; a CUDA-graph replay equals the eager call."""
    from posecnn_b200 import rescale
    B = 3
    I = _inputs(B, H, W, seed=H + W)
    out = _run_all(rescale, I, s, cuda)
    Ho, Wo = ref.scaled_size(H, W, s)
    assert out["color"].shape == (B, Ho, Wo, 3) and out["d16"].dtype == torch.uint16 and out["d32"].dtype == torch.float32
    host = {k: (v.view(torch.int16) if v.dtype == torch.uint16 else v).cpu().numpy() for k, v in out.items()}
    host["d16"] = host["d16"].view(np.uint16)
    for b in range(B):
        same_bits(host["color"][b], ref.color_blob(I["frames"][b], s))
        same_bits(host["x3"][b], ref.resize_linear_f32(I["x3"][b], s))
        same_bits(host["x1"][b], ref.resize_linear_f32(I["x1"][b], s))
        same_bits(host["d16"][b], ref.resize_linear_u16(I["depth"][b], s))
        same_bits(host["d32"][b], ref.resize_linear_u16(I["depth"][b], s).astype(np.float32))
        same_bits(host["label"][b], ref.resize_nearest(I["label"][b], s))
    if s == 1.0:
        same_bits(host["x3"], I["x3"])
        same_bits(host["d16"], I["depth"])
        same_bits(host["label"], I["label"])
    shard = _run_all(rescale, {k: v[1:2] for k, v in I.items()}, s, cuda)
    for k in out:
        assert torch.equal(ints(shard[k]), ints(out[k][1:2])), k
    static = {k: T(v, cuda) if k != "depth" else u16(v, cuda) for k, v in I.items()}

    def graphed():
        return dict(color=rescale.color_blob(static["frames"], s), x3=rescale.resize_linear(static["x3"], s),
                    d16=rescale.resize_depth(static["depth"], s), label=rescale.resize_nearest(static["label"], s))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graphed()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = graphed()
    g.replay()
    torch.cuda.synchronize()
    for k in cap:
        assert torch.equal(ints(cap[k]), ints(out[k])), k


def test_labels_back_to_the_frame(cuda):
    """test.py:1421: the 720 x 960 label map back to 480 x 640 at fx = 1 / 1.5."""
    from posecnn_b200 import rescale
    lab = np.random.default_rng(4).integers(0, 3, (2, 720, 960)).astype(np.int32)
    got = rescale.resize_nearest(T(lab, cuda), 1.0 / S).cpu().numpy()
    assert got.shape == (2, 480, 640)
    for b in range(2):
        same_bits(got[b], ref.resize_nearest(lab[b], 1.0 / S))


def test_training_inputs_follow_the_data_layer(cuda):
    """minibatch.py:179-183 (blob - PIXEL_MEANS, then LINEAR), :352 (label NEAREST), :416 (vertmap LINEAR), :435 (im_scale * center)
    restated with the numpy resize, per image, against training_inputs on the batch."""
    from posecnn_b200 import augment, rescale
    B, H, W, C = 2, 480, 640, 2
    sc = synth.make_coordinate_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=1, seed=12)
    rgb, _ = synth.make_images(B, H, W, seed=3)
    rgba = np.concatenate([rgb, np.full((B, H, W, 1), 255, np.uint8)], 3)
    params, keys = augment.draw_params(np.random.RandomState(4), B, 0, device=cuda)
    blob = augment.augment_color(T(rgba, cuda), None, params, keys)
    cen = np.zeros((B, C, 3), np.float32)
    cen[:, 1] = np.array([[311.37, 207.91, 0.83], [150.5, 333.25, 1.1]], np.float32)
    out = rescale.training_inputs(blob, T(sc["label"], cuda), T(cen, cuda), S, vertmap=T(sc["coords"], cuda))
    assert set(out) == {"data", "gt_label_2d", "centers", "vertmap"}
    blob_np = blob.cpu().numpy()
    for b in range(B):
        same_bits(out["data"][b].cpu().numpy(), ref.resize_linear_f32(blob_np[b], S))
        same_bits(out["gt_label_2d"][b].cpu().numpy(), ref.resize_nearest(sc["label"][b], S))
        same_bits(out["vertmap"][b].cpu().numpy(), ref.resize_linear_f32(sc["coords"][b], S))
    want_c = cen.copy()
    want_c[..., :2] = S * cen[..., :2]                      # float32 products, as numpy's im_scale * center
    same_bits(out["centers"].cpu().numpy(), want_c)
    assert rescale.training_inputs(blob, T(sc["label"], cuda), T(cen, cuda), S)["vertmap"] is None


# ---------------------------------------------------------------------------------------------------------------------
# the existing kernels at 720 x 960
# ---------------------------------------------------------------------------------------------------------------------
def _conv_cases():
    from tests.test_conv_gpu import _network_conv_cases
    return [c for c in _network_conv_cases(720, 960)]


def _wgrad_cases():
    from tests.test_backward_gpu import _wgrad_cases as cases
    return cases(720, 960)


_CONV, _WG = _conv_cases(), _wgrad_cases()


@pytest.mark.parametrize("name,H,W,Cin,Cout,k,pool,dgrad", _CONV, ids=[c[0] for c in _CONV])
def test_conv_exact_at_720x960(cuda, name, H, W, Cin, Cout, k, pool, dgrad):
    """test_conv_gpu.py::test_conv_exact_at_network_shapes at the 720 x 960 layer shapes (conv5 at 45 x 60, the heads at 90 x 120):
    integer operands, bit-exact, at least three work items per CTA."""
    from tests.test_conv_gpu import test_conv_exact_at_network_shapes as exact
    exact(cuda, name, H, W, Cin, Cout, k, pool, dgrad)


@pytest.mark.parametrize("name,H,W,Cin,Cout,k", _WG, ids=[c[0] for c in _WG])
def test_conv_wgrad_exact_at_720x960(cuda, name, H, W, Cin, Cout, k):
    """test_backward_gpu.py::test_conv_wgrad_exact_at_training_shapes at the 720 x 960 layer shapes."""
    from tests.test_backward_gpu import test_conv_wgrad_exact_at_training_shapes as exact
    exact(cuda, name, H, W, Cin, Cout, k)


def test_conv1_above_2_31_elements_equals_its_halves(cuda):
    """Batch 50 at 720 x 960: conv1_1's and conv1_2's activations hold 2.2e9 elements, past int32 flat indices.  conv1_1 (fused
    loader), conv1_2 and conv1_2 + pool1 on the whole batch equal the same calls on the two batch-25 halves bit for bit."""
    from posecnn_b200 import conv
    B, H, W = 50, 720, 960
    assert B * H * W * 64 > 2 ** 31
    g = torch.Generator(device=cuda).manual_seed(3)
    img = torch.randint(0, 256, (B, H, W, 3), generator=g, device=cuda, dtype=torch.uint8)
    w1 = conv.conv1_1_weights_to_tc(torch.randn(3, 3, 3, 64, generator=g, device=cuda) * 0.1)
    w2 = conv.hwio_to_tc(torch.randn(3, 3, 64, 64, generator=g, device=cuda) * 0.05)
    b1, b2 = torch.randn(64, generator=g, device=cuda) * 0.1, torch.randn(64, generator=g, device=cuda) * 0.1
    mean = (102.9801, 115.9465, 122.7717)
    a1 = conv.conv1_fused(img, w1, b1, mean, True)
    for lo, hi in ((0, 25), (25, 50)):
        assert torch.equal(conv.conv1_fused(img[lo:hi].contiguous(), w1, b1, mean, True).view(torch.int16), a1[lo:hi].view(torch.int16))
    del img
    for pool in (False, True):
        f = conv.conv_pool_bf16 if pool else conv.conv_bf16
        whole = f(a1, w2, b2, 3, True)
        for lo, hi in ((0, 25), (25, 50)):
            half = f(a1[lo:hi].contiguous(), w2, b2, 3, True)
            assert torch.equal(half.view(torch.int16), whole[lo:hi].view(torch.int16)), (pool, lo)
        del whole, half
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the C = 2 object-coordinate network at 720 x 960
# ---------------------------------------------------------------------------------------------------------------------
def test_coord_network_forward_720x960(cuda):
    """The vertex_reg_3d C = 2 network on color_blob(480 x 640 frames, 1.5): trunk, labels and vertex_pred against the fp32
    restatement with test_single_class_gpu.py::test_inference_two_classes_480x640's limits."""
    from posecnn_b200 import rescale
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from tests import ref_network as R
    C, B = 2, 2
    net = vgg16_convs(num_classes=C, device=cuda, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False,
                      scales=(S,)).init_random(seed=0)
    rgb, _ = synth.make_images(B, 480, 640, seed=3)
    data = rescale.color_blob(T(rgb, cuda), S)
    assert data.shape == (B, 720, 960, 3)
    meta = T(np.stack([synth.make_meta(synth.intrinsics(720, 960))] * B), cuda)
    ext = T(synth.extents_for(C), cuda)
    net.calibrate_background(data, meta, ext, 0.75)
    out = net.forward(data, meta, ext, want_prob=True)
    torch.cuda.synchronize()
    x = data.permute(0, 3, 1, 2)
    with torch.no_grad():
        feats = R.trunk(net.params, x)
        e = {n: rel_l2(out[n].float().permute(0, 3, 1, 2), feats[n]) for n in ("conv4_3", "conv5_3")}
        assert out["conv5_3"].shape[1:3] == (45, 60)
        score, label, prob, vertex = R.heads(net.params, feats["conv4_3"], feats["conv5_3"], C)
    ev = rel_l2(out["vertex_pred"].permute(0, 3, 1, 2), vertex)
    top2 = torch.topk(score, 2, dim=1).values
    decided = (top2[:, 0] - top2[:, 1]) / top2[:, 0].abs().clamp(min=1e-6) > 0.05
    frac = decided.float().mean().item()
    flips = (out["label_2d"][decided] != label[decided]).float().mean().item()
    print(f"720 x 960, C = 2: conv4_3 rel-L2 {e['conv4_3']:.2e}, conv5_3 {e['conv5_3']:.2e}; vertex rel-L2 {ev:.2e}; {frac:.3f} "
          f"decided by > 5 %, flip rate there {flips:.2e}")
    assert max(e.values()) < 2e-2 and ev < 2e-2 and frac > 0.2 and flips < 1e-3
    assert torch.allclose(out["prob_normalized"].sum(3), torch.ones_like(out["prob_normalized"][..., 0]), atol=1e-5)


def test_coord_training_step_720x960(cuda):
    """Trainer.step at 720 x 960, batch 2 (IMS_PER_BATCH of the LINEMOD configurations), on training_inputs of a 480 x 640 scene:
    every gradient against the 16-bit-rounded and the pure fp32 autograd graph within test_train_coord_gpu.py's limits_coord(2)."""
    from posecnn_b200 import rescale
    from posecnn_b200.networks.vgg16_convs import PIXEL_MEANS
    from posecnn_b200.train import Trainer
    from tests.test_train_coord_gpu import coord_scene, limits_coord, make_coord_net
    from tests.train_coord_ref import coord_reference_grads, vertex_targets_3d
    from tests.train_ref import compare_grads
    C, B, vw_, wi = 2, 2, 10.0, 10.0
    rgb, _ = synth.make_images(B, 480, 640, seed=3)
    sc, cen = coord_scene(B, 480, 640, C, seed=11)
    blob = (T(rgb, cuda).float() - torch.tensor(PIXEL_MEANS, device=cuda, dtype=torch.float64)).float()
    I = rescale.training_inputs(blob, T(sc["label"], cuda), T(cen, cuda), S, vertmap=T(sc["coords"], cuda))
    meta = T(np.stack([synth.make_meta(synth.intrinsics(720, 960)).reshape(48)] * B), cuda)
    args = (I["data"], I["gt_label_2d"], I["centers"], meta, T(sc["extents"], cuda), torch.zeros((0, 13), device=cuda),
            T(synth.make_model_points(C, 50), cuda), torch.zeros(C, device=cuda))
    vm = I["vertmap"]
    net = make_coord_net(cuda, C)
    tr = Trainer(net, lr=0.01, vertex_w=vw_, vertex_w_inside=wi)
    A = tr.forward(*args, vertmap=vm)
    grads = tr.backward(A, args[1], args[2], vertmap=vm)
    torch.cuda.synchronize()
    vt, vwt = vertex_targets_3d(args[1].cpu().numpy(), vm.cpu().numpy(), args[2].cpu().numpy(), args[4].cpu().numpy(), wi)
    assert vwt.any()
    ref_args = (I["data"] + torch.tensor(PIXEL_MEANS, device=cuda),) + args[1:]     # the reference subtracts the means itself
    P, r16 = coord_reference_grads(net, ref_args, (vt, vwt), True, vw_)
    Pf, r32 = coord_reference_grads(net, ref_args, (vt, vwt), False, vw_)
    ev = rel_l2(tr.dense_vertex_pred(A).permute(0, 3, 1, 2), r16["vertex"])
    print(f"720 x 960, C = 2: loss_vertex {vw_ * A['vtx_out'][0].item():.5f} (16-bit-rounded graph {r16['loss_vertex']:.5f}, fp32 "
          f"{r32['loss_vertex']:.5f}); loss_cls {A['cls_out'][0].item():.5f} ({r16['loss_cls']:.5f}); vertex_pred rel-L2 {ev:.2e}")
    assert ev < 1e-2
    for r_ in (r16, r32):
        assert abs(A["cls_out"][0].item() - r_["loss_cls"]) < 3e-2 * max(1.0, abs(r_["loss_cls"]))
        assert abs(vw_ * A["vtx_out"][0].item() - r_["loss_vertex"]) < 3e-2 * max(1.0, abs(r_["loss_vertex"]))
    compare_grads(tr, grads, P, Pf, sorted(grads), limits_coord(C))


# ---------------------------------------------------------------------------------------------------------------------
# the test-time flow on a planted scene
# ---------------------------------------------------------------------------------------------------------------------
def test_planted_scene_through_the_scaled_test_flow(cuda):
    """An analytic 480 x 640 scene (two images, one object each) resized as the test path does (labels NEAREST, the object's
    coordinates LINEAR, uint16 depth LINEAR, K * 1.5): estimate_poses_3d and ICP on the 720 x 960 maps recover the planted poses
    (ICP's rotation about an ellipsoid's symmetry axis is not observable and is not scored); estimate_poses_2d equals the float64
    restatement on the same maps, and its error against the planted pose is printed: its survivor keeps the P3P pose of four
    pixels (no refit, as the reference), so the resampled coordinates of those four pixels decide it.  The records' boxes are in
    720 x 960 pixels; the labels return to 480 x 640."""
    from posecnn_b200 import rescale
    from posecnn_b200.coord_pose import assemble_records, estimate_poses_2d, estimate_poses_3d
    from posecnn_b200.pose_refine import refine_poses
    from tests import coord_pose2d_ref as ref2
    from tests.test_coord_pose_cpu import PLANTED_ROT_DEG, PLANTED_TRANS_M, rot_err_deg
    from tests.test_pose_refine_cpu import observable_rot_err_deg
    C, B = 2, 2
    sc = synth.make_coordinate_scene(batch=B, num_classes=C, objects_per_image=1, seed=8)
    label = rescale.resize_nearest(T(sc["label"], cuda), S)
    vert = rescale.resize_linear(T(np.ascontiguousarray(sc["vertex"][..., 3:6]), cuda), S)
    vertex = torch.cat([torch.zeros_like(vert), vert], 3).contiguous()
    depth = rescale.resize_depth(T(np.rint(sc["depth"]).astype(np.float32), cuda), S)
    meta = T(np.stack([synth.make_meta(synth.intrinsics(720, 960))] * B), cuda)
    ext = T(sc["extents"], cuda)
    keys = torch.tensor([5, 6], dtype=torch.int64, device=cuda)
    meta_np = meta.cpu().numpy()
    assert label.shape == depth.shape == (B, 720, 960)
    e3 = estimate_poses_3d(label, depth, meta, ext, keys, vertex=vertex)
    e2 = estimate_poses_2d(label, meta, ext, keys, vertex=vertex)
    rois, poses, num = assemble_records(e3["poses"], ext, meta, S)
    assert int(num.item()) == B
    icp = refine_poses(label, depth, meta, torch.nn.functional.pad(rois, (0, 1)), poses, T(sc["points"][:C], cuda), num_rows=num)
    p3, p2, q_icp = e3["poses"].cpu().numpy(), e2["poses"].cpu().numpy(), icp["poses_icp"].cpu().numpy()
    r = rois.cpu().numpy()
    lab = label.cpu().numpy()
    worst = dict(rot3=0.0, t3=0.0, rot2=0.0, t2=0.0, rot_icp=0.0, t_icp=0.0)
    for k, row in enumerate(sc["poses"]):
        b, c = int(row[0]), int(row[1])
        R, t = synth.quat_to_rot(row[2:6]), row[6:9]
        for tag, P in (("3", p3[b, c]), ("2", p2[b, c])):
            worst["rot" + tag] = max(worst["rot" + tag], rot_err_deg(P[:, :3].astype(np.float64), R))
            worst["t" + tag] = max(worst["t" + tag], float(np.linalg.norm(P[:, 3] - t)))
        worst["rot_icp"] = max(worst["rot_icp"], observable_rot_err_deg(q_icp[k, :4], row[2:6], sc["extents"][c]))
        worst["t_icp"] = max(worst["t_icp"], float(np.linalg.norm(q_icp[k, 4:] - t)))
        # the box is in 720 x 960 pixels: it holds the scaled object mask
        ys, xs = np.nonzero(lab[b] == c)
        assert r[k, 0] == b and r[k, 1] == c
        assert r[k, 2] <= xs.min() + 2 and r[k, 3] <= ys.min() + 2 and r[k, 4] >= xs.max() - 2 and r[k, 5] >= ys.max() - 2, r[k]
    print(f"planted at 720 x 960: {worst}")
    assert worst["rot3"] < PLANTED_ROT_DEG and worst["t3"] < PLANTED_TRANS_M
    vert_np, lab_np = vertex.cpu().numpy(), lab
    for b in range(B):
        want = ref2.estimate_image(lab_np[b], vert_np[b], sc["extents"], tuple(meta_np[b, [0, 4, 2, 5]]), 5 + b, C)
        assert e2["info"][b, 1, 5].item() == want["info"][1, 5]                     # the same survivor
        assert np.abs(p2[b, 1] - want["poses"][1]).max() < 1e-4, (p2[b, 1], want["poses"][1])
    assert worst["rot_icp"] < PLANTED_ROT_DEG and worst["t_icp"] < PLANTED_TRANS_M
    frame = rescale.resize_nearest(label, 1.0 / S).cpu().numpy()
    assert frame.shape == sc["label"].shape
    for b in range(B):
        same_bits(frame[b], ref.resize_nearest(lab[b], 1.0 / S))
        inter = ((frame[b] > 0) & (sc["label"][b] > 0)).sum()
        union = ((frame[b] > 0) | (sc["label"][b] > 0)).sum()
        assert inter / union > 0.97, inter / union
