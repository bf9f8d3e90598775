"""Object-coordinate (VERTEX_REG_3D) training on the GPU: the materialised 3-D targets against the reference's own lines, the fused
loss (dense and 1/8-resolution sources) against smooth_l1_loss_vertex on the materialised blobs, the up-sampling adjoint's 3-D mode
against torch, the training step against the autograd graph, its contents, a short training run whose weights then estimate poses
on an inference network, and two ranks.  Every measured error is printed."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from posecnn_b200 import synth
from tests.test_train_coord_cpu import load_golden
from tests.train_coord_ref import vertex_targets_3d
from tests.train_ref import bits, compare_grads, limits, rel_l2, run_two_ranks

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def limits2(name):
    """test_single_class_gpu.limits2: train_ref.limits(), except conv2_x, which takes conv1_x's limits at C = 2."""
    return limits("conv1_2/w" if name.startswith("conv2_") else name)


def limits_coord(C):
    """train_ref.limits (C = 6) / limits2 (C = 2), except conv2_x .. conv4_x, held to at least 0.1 / 0.15 (16-bit-rounded / pure fp32
    graph).  With VERTEX_W 10 and a 3-D target the random network is far from (loss_vertex ~76 against loss_cls ~8), the trunk's
    gradient is the vertex branch's, and its smooth L1 sits in the L1 regime: a dense field of +-w_inside per labelled channel with
    none of the cancellation the 2-D step's gradients have.  The bf16 rounding of that propagated gradient then shows amplified
    from conv4_x down, as limits() describes for conv1_x.  Measured (B = 2, 64 x 96): at C = 6, 5.3e-2 .. 7.7e-2 / 7.4e-2 .. 0.110
    on conv2_1 .. conv4_2 (conv2_2/w largest); at C = 2, conv3_1 7.0e-2 / 0.119.  Every other parameter stays within the 2-D
    step's limits (vertex heads 1.8e-2 / 6.6e-3 at C = 6)."""
    base = limits2 if C == 2 else limits

    def lim(name):
        l16, l32 = base(name)
        if name[:5] in ("conv2", "conv3", "conv4"):
            l16, l32 = max(l16, 0.1), max(l32, 0.15)
        return l16, l32
    return lim


def coord_scene(B, H, W, C, seed, drop_one=True):
    """Labels, vertmap (unscaled object coordinates) and extents of make_coordinate_scene, and the presence table `centers` of the
    placed objects; with drop_one, image 0's first object is not listed (its pixels keep their label but get no target)."""
    sc = synth.make_coordinate_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=3 if C > 2 else 1, seed=seed)
    cen = np.zeros((B, C, 3), np.float32)
    for row in sc["poses"]:
        cen[int(row[0]), int(row[1])] = (0.0, 0.0, row[8])
    if drop_one:
        cen[0, int(sc["poses"][0][1]), 2] = 0.0
    return sc, cen


# ---------------------------------------------------------------------------------------------------------------------
# 1. materialised targets
# ---------------------------------------------------------------------------------------------------------------------
def test_targets_3d_equal_reference_golden(cuda):
    from posecnn_b200 import train_ops
    g, cen = load_golden()
    t, w = train_ops.generate_vertex_targets_3d(T(g["label"], cuda), T(g["vertmap"], cuda), T(cen, cuda), T(g["extents"], cuda),
                                                float(g["w_inside"]))
    t, w = t.cpu().numpy(), w.cpu().numpy()
    assert np.array_equal(t.view(np.int32), g["targets"].view(np.int32))
    assert np.array_equal(w, g["weights"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. fused loss
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [2, 22])
def test_fused_coord_loss_equals_materialised(cuda, C):
    """vertex_loss_from_coords (dense vertex_pred, with gradient; and the 1/8-resolution source) == smooth_l1_loss_vertex on the
    materialised blobs: loss within 1e-6 relative, gradient identical; dense and low-resolution sources bit-identical."""
    from posecnn_b200 import train_ops
    from posecnn_b200._lib import check, lib, ptr, stream
    B, H, W = 2, 240, 320
    sc, cen = coord_scene(B, H, W, C, seed=31)
    g = torch.Generator().manual_seed(C)
    lowres = (torch.randn(B, H // 8, W // 8, 4 * C, generator=g) * 0.5).to(cuda)
    bs, bv = torch.zeros(C, device=cuda), (torch.randn(3 * C, generator=g) * 0.1 + 0.5).to(cuda)
    label = torch.empty((B, H, W), dtype=torch.int32, device=cuda)
    vertex = torch.empty((B, H, W, 3 * C), device=cuda)
    check(lib().pcnn_up8_heads(ptr(lowres), ptr(bs), ptr(bv), B, H // 8, W // 8, C, ptr(label), ptr(vertex), ptr(None), ptr(None), stream()))
    lab, vm, cn, ext = T(sc["label"], cuda), T(sc["coords"], cuda), T(cen, cuda), T(sc["extents"], cuda)
    for sigma in (1.0, 2.5):
        vt, vw = train_ops.generate_vertex_targets_3d(lab, vm, cn, ext, 10.0)
        l0, w0, g0 = train_ops.smooth_l1_loss_vertex(vertex, vt, vw, sigma, want_grad=True, upstream=0.7)
        l1, w1, g1 = train_ops.vertex_loss_from_coords(vertex, lab, vm, cn, ext, 10.0, sigma, want_grad=True, upstream=0.7)
        l2, w2 = train_ops.vertex_loss_from_coords(lowres, lab, vm, cn, ext, 10.0, sigma, bias_vertex=bv)
        torch.cuda.synchronize()
        print(f"C = {C}, sigma {sigma}: sum w {w0.item():.0f}, loss {l0.item():.6f} materialised / {l1.item():.6f} fused "
              f"(rel {abs(l0.item() - l1.item()) / abs(l0.item()):.2e})")
        assert float(w0.item()) == float(w1.item()) == float(w2.item()) > 0
        assert abs(float(l0.item()) - float(l1.item())) <= 1e-6 * abs(float(l0.item()))
        assert torch.equal(g0, g1)
        assert float(l1.item()) == float(l2.item())
    # the unlisted object's pixels carry no weight
    c0 = int(sc["poses"][0][1])
    assert (sc["label"][0] == c0).any() and not bool(vw[0, ..., 3 * c0:3 * c0 + 3].any())


# ---------------------------------------------------------------------------------------------------------------------
# 3. the up-sampling adjoint's 3-D mode
# ---------------------------------------------------------------------------------------------------------------------
def _up8_problem(cuda, B, h, w, C, seed):
    from posecnn_b200._lib import check, lib, ptr, stream
    g = torch.Generator().manual_seed(seed)
    H, W = 8 * h, 8 * w
    lowres = (torch.randn(B, h, w, 4 * C, generator=g) * 0.7).to(cuda)
    bs, bv = (torch.randn(C, generator=g) * 0.1).to(cuda), (torch.randn(3 * C, generator=g) * 0.1 + 0.5).to(cuda)
    vertex = torch.empty((B, H, W, 3 * C), device=cuda)
    label = torch.empty((B, H, W), dtype=torch.int32, device=cuda)
    prob, score = torch.empty((B, H, W, C), device=cuda), torch.empty((B, H, W, C), device=cuda)
    check(lib().pcnn_up8_heads(ptr(lowres), ptr(bs), ptr(bv), B, h, w, C, ptr(label), ptr(vertex), ptr(prob), ptr(score), stream()))
    gt = torch.randint(-1, C, (B, H, W), generator=g).to(torch.int32)
    gt[:, : H // 4] = 0
    gt[:, H // 4: H // 2, : W // 2] = 1 if C == 2 else 2
    ext = (torch.rand(C, 3, generator=g) * 0.25 + 0.03)
    ext[0] = 0.0
    ext[1, 2] = 0.0                                            # a zero-extent axis: target 0 there
    vm = ((torch.rand(B, H, W, 3, generator=g) - 0.5) * 0.3)
    cen = torch.zeros(B, C, 3)
    cen[0, 1:, 2] = 1.0                                        # image 0 lists every class
    cen[1, 1:C:2, 2] = 1.0 if C > 2 else 0.0                   # image 1 every other class (none at C = 2)
    return dict(lowres=lowres, bv=bv, vertex=vertex, prob=prob, score=score, gt=gt.to(cuda), centers=cen.to(cuda), ext=ext.to(cuda),
                vertmap=vm.to(cuda), B=B, h=h, w=w, C=C)


def _up8_bwd(P, dense, coord, thr=0.7, up_vtx=2.0, w_in=10.0, count=937.0, sumw=411.0):
    from posecnn_b200._lib import check, lib, ptr, stream
    B, h, w, C = P["B"], P["h"], P["w"], P["C"]
    dev = P["lowres"].device
    d_sc = torch.full((B, h, w, 64), 7.0, dtype=torch.bfloat16, device=dev)             # padding channels must be written as 0
    d_vt = torch.full((B, h, w, 128), 7.0, dtype=torch.bfloat16, device=dev)
    dbias = torch.empty((4 * C,), device=dev)
    cls_out, vtx_out = torch.tensor([0.5, count], device=dev), torch.tensor([0.25, sumw], device=dev)
    ws = torch.empty(4 * B * ((w + 3) // 4) * ((h + 15) // 16) * 4 * C, dtype=torch.uint8, device=dev)
    src = (ptr(P["vertex"] if dense else None), ptr(None if dense else P["lowres"]), ptr(None if dense else P["bv"]))
    head = (ptr(P["prob"]), ptr(P["score"]), ptr(P["gt"]), ptr(cls_out), 1.0, thr) + src
    tail = (ptr(vtx_out), up_vtx, w_in, 1.0, B, h, w, C, 64, 128, ptr(d_sc), ptr(d_vt), ptr(dbias), ptr(ws),
            ws.numel(), stream())
    if coord:
        check(lib().pcnn_up8_heads_bwd_coord(*head, ptr(P["vertmap"]), ptr(P["centers"]), ptr(P["ext"]), *tail))
    else:
        check(lib().pcnn_up8_heads_bwd_ex(*head, ptr(P["centers"]), *tail))
    return d_sc, d_vt, dbias


@pytest.mark.parametrize("C", [2, 6, 22])
@pytest.mark.parametrize("h,w", [(18, 10), (60, 80)])
def test_up8_backward_coord_against_torch(cuda, C, h, w):
    """The method of test_single_class_gpu.py::test_up8_backward_two_classes_against_torch with the 3-D target: d_vt within 4e-3
    relative-L2 of torch, d_sc byte-identical to the 2-D entry's on the same inputs, dense == low-resolution source, two launches
    bit-identical."""
    B, thr, up_vtx, w_in, count, sumw = 2, 0.7, 2.0, 10.0, 937.0, 411.0
    P = _up8_problem(cuda, B, h, w, C, seed=h * 100 + w + C)
    d_sc, d_vt, dbias = _up8_bwd(P, True, True)
    e_sc, e_vt, ebias = _up8_bwd(P, False, True)
    again = _up8_bwd(P, False, True)
    s2d = _up8_bwd(P, False, False)
    torch.cuda.synchronize()
    for a, b in zip((e_sc, e_vt, ebias), again):
        assert torch.equal(bits(a), bits(b))
    assert torch.equal(bits(d_sc), bits(e_sc)) and torch.equal(bits(d_vt), bits(e_vt)) and torch.equal(bits(dbias), bits(ebias))
    assert torch.equal(bits(e_sc), bits(s2d[0]))
    assert torch.equal(bits(ebias[:C]), bits(s2d[2][:C]))
    H, W = 8 * h, 8 * w
    gt = P["gt"].long()
    g0 = gt.clamp(min=0)
    vertex = P["vertex"]
    # the 3-D target from the materialised restatement (float32 numpy, bit-exact to the device's: test_targets_3d_equal_reference_golden)
    tg_np, wt_np = vertex_targets_3d(P["gt"].cpu().numpy(), P["vertmap"].cpu().numpy(), P["centers"].cpu().numpy(), P["ext"].cpu().numpy(), 1.0)
    tg, wt = torch.from_numpy(tg_np).to(cuda), torch.from_numpy(wt_np).to(cuda)
    assert bool(wt[0].any())
    diff = w_in * (vertex - tg)
    dt = torch.where(diff.abs() < 1.0, diff, diff.sign())
    d_up_v = (up_vtx / (sumw + 1e-10)) * w_in * dt * wt
    prob, score = P["prob"], P["score"]
    pg = prob.gather(3, g0[..., None])[..., 0]
    sel = (gt >= 0) & ((gt > 0) | (pg < thr))
    d_up_s = (1.0 / (count + 1e-10)) * sel[..., None] * (prob - F.one_hot(g0, C).float()) * (score > 0)
    d_up = torch.cat([d_up_s, d_up_v], 3).permute(0, 3, 1, 2).contiguous()
    k1 = torch.tensor([1.0 - abs(i / 8.0 - 0.9375) for i in range(16)], device=cuda)
    filt = (k1[:, None] * k1[None, :])[None, None].expand(4 * C, 1, 16, 16).contiguous()
    want = F.conv2d(d_up, filt, stride=8, padding=4, groups=4 * C).permute(0, 2, 3, 1)
    ev = rel_l2(d_vt[..., :3 * C].float(), want[..., C:])
    print(f"C = {C}, h, w = {h}, {w}: d_vt rel-L2 {ev:.2e}; max |dbias - torch| {(dbias - d_up.sum((0, 2, 3))).abs().max().item():.2e}")
    assert ev < 4e-3
    assert (d_vt[..., 3 * C:].float() == 0).all() and (d_sc[..., C:].float() == 0).all()
    assert torch.allclose(dbias, d_up.sum((0, 2, 3)), rtol=2e-4, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the training step
# ---------------------------------------------------------------------------------------------------------------------
def make_coord_net(cuda, C, pose_reg=False, seed=0):
    """tests/train_ref.make_net for an object-coordinate network."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(num_classes=C, device=cuda, is_train=True, fold_vertex_head=False, vertex_reg_2d=False, vertex_reg_3d=True,
                      pose_reg=pose_reg).init_random(seed=seed, bias_std=0.02)
    net.params["score/weights"] *= 0.02
    net.params["vertex_pred/weights"] *= 0.02
    net.prepare()
    return net


def coord_inputs(cuda, C, B=2, H=64, W=96, seed=11):
    """(args, vertmap): Trainer.step's positional inputs (data, gt_label_2d, centers, meta_data, extents, gt_poses, points,
    symmetry) with labels, presence table and extents of a coordinate scene, and its object-coordinate map."""
    rgb, _ = synth.make_images(B, H, W, seed=3)
    sc, cen = coord_scene(B, H, W, C, seed)
    meta = np.stack([synth.make_meta(synth.intrinsics(H, W)).reshape(48)] * B)
    args = (T(rgb, cuda), T(sc["label"], cuda), T(cen, cuda), T(meta, cuda), T(sc["extents"], cuda), torch.zeros((0, 13), device=cuda),
            T(synth.make_model_points(C, 50), cuda), torch.zeros(C, device=cuda))
    return args, T(sc["coords"], cuda)


def _coord_grads(tr, args, vertmap):
    A = tr.forward(*args, vertmap=vertmap)
    g = tr.backward(A, args[1], args[2], vertmap=vertmap)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in g.items()}


@pytest.mark.parametrize("C", [6, 2])
def test_training_step_coord(cuda, C):
    """VERTEX_W 10: every gradient against the 16-bit-rounded and the pure fp32 autograd graph of the object-coordinate network
    (tests/train_coord_ref.coord_reference_grads on the 3-D targets) within limits_coord(C)."""
    from posecnn_b200.train import Trainer
    from tests.train_coord_ref import coord_reference_grads
    vw_, wi = 10.0, 10.0
    net = make_coord_net(cuda, C)
    args, vm = coord_inputs(cuda, C)
    tr = Trainer(net, lr=0.01, vertex_w=vw_, vertex_w_inside=wi)
    A = tr.forward(*args, vertmap=vm)
    grads = tr.backward(A, args[1], args[2], vertmap=vm)
    torch.cuda.synchronize()
    assert set(grads) == set(tr.master)
    vt, vwt = vertex_targets_3d(args[1].cpu().numpy(), vm.cpu().numpy(), args[2].cpu().numpy(), args[4].cpu().numpy(), wi)
    assert vwt.any()
    P, ref = coord_reference_grads(net, args, (vt, vwt), True, vw_)
    Pf, reff = coord_reference_grads(net, args, (vt, vwt), False, vw_)
    ev = rel_l2(tr.dense_vertex_pred(A).permute(0, 3, 1, 2), ref["vertex"])
    print(f"C = {C}: loss_vertex {vw_ * A['vtx_out'][0].item():.5f} (16-bit-rounded graph {ref['loss_vertex']:.5f}, fp32 "
          f"{reff['loss_vertex']:.5f}); loss_cls {A['cls_out'][0].item():.5f} ({ref['loss_cls']:.5f}); vertex_pred rel-L2 {ev:.2e}")
    assert ev < 1e-2
    for r_ in (ref, reff):
        assert abs(A["cls_out"][0].item() - r_["loss_cls"]) < 3e-2 * max(1.0, abs(r_["loss_cls"]))
        assert abs(vw_ * A["vtx_out"][0].item() - r_["loss_vertex"]) < 3e-2 * max(1.0, abs(r_["loss_vertex"]))
    compare_grads(tr, grads, P, Pf, sorted(grads), limits_coord(C))


def test_step_contents_coord(cuda):
    """No fc state; step() returns loss_cls, loss_vertex, loss and grads; pose_reg=True on a 3-D network steps exactly like
    pose_reg=False (the score / vertex_pred bias sums are held to the run-to-run spread, as the pose_reg=False test does);
    vertmap is required."""
    from posecnn_b200.train import Trainer
    C = 6
    args, vm = coord_inputs(cuda, C)
    trs = [Trainer(make_coord_net(cuda, C, pose_reg=p), lr=0.01, vertex_w=10.0) for p in (False, True)]
    for tr in trs:
        assert tr.coord and not tr.pose_reg and tr.fc_t == {}
        for d in (tr.master, tr.accum, tr.tc):
            assert not any(k.startswith(("fc6", "fc7", "fc8", "fc9")) for k in d)
    with pytest.raises(ValueError, match="vertmap"):
        trs[0].forward(*args)
    a, a2, b = _coord_grads(trs[0], args, vm), _coord_grads(trs[0], args, vm), _coord_grads(trs[1], args, vm)
    unfixed = {k for k in a if not torch.equal(a[k], a2[k])}
    print("run-to-run differences:", sorted(unfixed))
    assert unfixed <= {"score/b", "vertex_pred/b"}
    assert set(a) == set(b)
    for k in a:
        if k in unfixed:
            assert torch.allclose(a[k], b[k], rtol=1e-5, atol=1e-9), k
        else:
            assert torch.equal(bits(a[k]), bits(b[k])), k
    outs = [tr.step(*args, vertmap=vm) for tr in trs]
    for out in outs:
        assert set(out) == {"loss_cls", "loss_vertex", "loss", "grads"}
        assert torch.isfinite(out["loss"]).all() and torch.allclose(out["loss"], out["loss_cls"] + out["loss_vertex"])
    assert torch.allclose(outs[0]["loss"], outs[1]["loss"], rtol=1e-6)
    A = trs[0].forward(*args, vertmap=vm)
    assert not any(k in A for k in ("rois", "pool", "fc6", "fc7", "poses_tanh", "loss_pose_raw", "num_rois"))


def test_training_lowers_loss_and_exported_weights_estimate_poses(cuda):
    """20 steps on one fixed batch lower loss_vertex; export_params() then loads into an inference network
    (vertex_reg_2d=False, vertex_reg_3d=True, is_train=False), whose forward(estimate_depth=...) runs.  The random network's
    gradients are large (trunk weight gradients ~1e3 in norm at VERTEX_W 10), so the run takes lr 1e-6 (1e-3 diverges in 3 steps)."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.train import Trainer
    C, B, H, W = 6, 2, 128, 160
    net = make_coord_net(cuda, C)
    args, vm = coord_inputs(cuda, C, B=B, H=H, W=W, seed=5)
    tr = Trainer(net, lr=1e-6, vertex_w=10.0, vertex_w_inside=10.0)
    hist = []
    for _ in range(20):
        out = tr.step(*args, vertmap=vm)
        hist.append((out["loss_vertex"].item(), out["loss_cls"].item()))
    print("loss_vertex:", " ".join(f"{v:.4f}" for v, _ in hist))
    print("loss_cls:   ", " ".join(f"{c:.4f}" for _, c in hist))
    assert all(np.isfinite(hist).flatten())
    assert hist[-1][0] < hist[0][0]
    tr.export_params()
    inf = vgg16_convs(num_classes=C, device=cuda, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False, is_train=False)
    inf.params = {k: v.clone() for k, v in net.params.items()}
    inf.prepare()
    assert torch.equal(inf.params["vertex_pred/biases"], tr.master["vertex_pred/b"])
    depth = torch.from_numpy(synth.make_images(B, H, W, seed=3)[1] * 10000.0).float().to(cuda)
    keys = torch.tensor([3, 9], dtype=torch.int64, device=cuda)
    o = inf.forward(args[0], args[3], args[4], dense_vertex=False, estimate_depth=depth, estimate_keys=keys)
    torch.cuda.synchronize()
    assert o["estimate_poses"].shape[0] == B and torch.isfinite(o["estimate_poses"]).all()
    assert o["detections_rois"].shape == (B * (C - 1), 6)
    print("estimate_info (image, class) sums:", o["estimate_info"].sum((0, 1)).tolist())


# ---------------------------------------------------------------------------------------------------------------------
# 5. two ranks
# ---------------------------------------------------------------------------------------------------------------------
COORD_WORKER = r'''
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
from posecnn_b200 import parallel
from posecnn_b200.train import Trainer
from tests.test_train_coord_gpu import coord_inputs, make_coord_net
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
B, C = 4, 6
(data, gt, cen, meta, ext, gtp, pts, sym), vm = coord_inputs(dev, C, B=B)
o, n = parallel.shard_range(B, rank, world)
single = Trainer(make_coord_net(dev, C), lr=0.01, vertex_w=10.0)
ref = single.step(data, gt, cen, meta, ext, gtp, pts, sym, vertmap=vm)
tr = Trainer(make_coord_net(dev, C), lr=0.01, vertex_w=10.0, world=world)
out = tr.step(data[o:o + n], gt[o:o + n], cen[o:o + n], meta[o:o + n], ext, gtp, pts, sym, vertmap=vm[o:o + n])
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
tot = torch.stack([out[k][0] for k in ("loss_cls", "loss_vertex")])
dist.all_reduce(tot)
want = torch.stack([ref[k][0] for k in ("loss_cls", "loss_vertex")])
assert torch.allclose(tot, want, rtol=1e-4, atol=1e-6), (tot, want)
dist.barrier()
dist.destroy_process_group()
print("COORD_RANK_OK", rank, worst)
'''


def test_two_rank_step_coord(tmp_path):
    """One object-coordinate step on image shards over 2 ranks == the step on the whole batch on one GPU (skips with fewer than
    2 GPUs)."""
    from tests.train_ref import ROOT
    run_two_ranks(tmp_path, COORD_WORKER % dict(root=ROOT), marker="COORD_RANK_OK")
