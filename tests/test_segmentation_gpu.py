"""The segmentation network on the device (vgg16_convs with vertex_reg_2d = vertex_reg_3d = False, lib/networks/vgg16_convs.py:79-149):
its score-only heads against a 2-D vertex network sharing the same parameters, the classification-only adjoint against the 2-D
adjoint with the vertex loss switched off, the training step against torch autograd of the segmentation graph, the inference
graph, image shards, Evaluator on its labels, and the two-rank step."""
import numpy as np
import pytest
import torch

from tests import heads_ref as R
from tests.seg_ref import make_seg_net, seg_reference_grads
from tests.train_ref import bits, compare_grads, depth_blob_np, make_inputs, run_two_ranks

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def _same(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bad = bits(a) != bits(b)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} differ; first at {bad.nonzero()[0].tolist()}"


def _vertex_twin(seg, cuda):
    """A 2-D vertex network (pose head, folded vertex head) whose trunk(s), score_conv4 / 5 and score are seg's."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(input_format=seg.input_format, num_classes=seg.num_classes, device=cuda).init_random(seed=1)
    for k in seg.param_shapes():
        net.params[k] = seg.params[k]
    net.prepare()
    return net


# ---------------------------------------------------------------------------------------------------------------------
# 1. score-only heads, forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [2, 8, 9, 10, 22])
def test_heads_match_the_vertex_network(cuda, C):
    """480 x 640, batch 4: label_2d, prob_normalized and score of the segmentation network are byte-identical to the 2-D network's
    on shared parameters, in the full mode (k_up8_heads) and on the label-only fast path (k_up8_label); C = 9 runs the one-channel-
    per-thread forms."""
    B, H, W = 4, 480, 640
    (data, _, _, meta, ext, _, _, _), _, _ = make_inputs(cuda, B=B, H=H, W=W, C=C)
    seg = make_seg_net(cuda, C=C, is_train=False, seed=C)
    two = _vertex_twin(seg, cuda)
    assert seg._tc.keys() < two._tc.keys()
    got = seg.forward(data, meta, ext, want_prob=True, want_score=True)
    want = two.forward(data, meta, ext, want_prob=True, want_score=True, sync_rois=False)
    torch.cuda.synchronize()
    assert set(got) == {"conv4_3", "conv5_3", "score_conv4", "score_conv5", "label_2d", "prob_normalized", "score"}
    assert seg._last_lowres.shape == (B, H // 8, W // 8, C)          # no vertex channel is computed or stored
    for k in ("label_2d", "prob_normalized", "score"):
        _same(got[k], want[k], k)
    labels = torch.bincount(got["label_2d"].flatten().long(), minlength=C)
    print(f"C={C}: {int((labels > 0).sum())} classes present in label_2d")
    assert int((labels > 0).sum()) >= 2
    lab = seg.forward(data, meta, ext)["label_2d"]
    lab2 = two.forward(data, meta, ext, dense_vertex=False, sync_rois=False)["label_2d"]
    torch.cuda.synchronize()
    _same(lab, lab2, "label_2d, label-only")
    _same(lab, got["label_2d"], "label_2d, label-only against the full mode")


def test_vertex_outputs_are_refused(cuda):
    (data, _, _, meta, ext, _, _, _), _, depth = make_inputs(cuda, B=1, H=64, W=96, C=10)
    seg = make_seg_net(cuda, C=10, is_train=False)
    for kw in (dict(dense_vertex=True), dict(estimate_depth=depth), dict(estimate_rgb=True), dict(refine_depth=depth)):
        with pytest.raises(ValueError, match="segmentation"):
            seg.forward(data, meta, ext, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the classification-only adjoint
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(60, 80), (37, 27)])
@pytest.mark.parametrize("C", [2, 8, 9, 10, 22])
def test_adjoint_matches_the_2d_mode(cuda, C, h, w):
    """d_sc and dbias[:C] of target mode "none" are byte-identical to pcnn_up8_heads_bwd's 2-D mode at upstream_vertex = 0, on 480 x 640
    (ragged last band) and 296 x 216 (a ragged last strip of the 4- and the 16-cell kernels); padding channels are written 0."""
    from posecnn_b200 import heads
    B = 2
    plan = R.up8_bwd_plan(B, h, w, C)
    if (h, w) == (37, 27):
        assert plan["last_strip_cells"] < plan["strip"]
    g = torch.Generator().manual_seed(500 * C + h)
    P = R.up8_bwd_problem(B, h, w, C, False, g, device=cuda)
    cls_out = torch.tensor([0.5, P["count"]], device=cuda)
    vtx_out = torch.tensor([0.25, P["sumw"]], device=cuda)
    for thr in (1.0, 0.5):
        d_sc, d_vt, dbias = heads.up8_heads_bwd(P["prob"], P["score"], P["gt"], cls_out, P["up_cls"], thr, P["lowres"], P["bias_v"],
                                                P["centers"], vtx_out, 0.0, P["w_inside"], 1.0)
        out = (torch.full((B, h, w, 64), 7.0, dtype=torch.bfloat16, device=cuda), torch.full((C,), 7.0, device=cuda))
        e_sc, ebias = heads.up8_scores_bwd(P["prob"], P["score"], P["gt"], cls_out, P["up_cls"], thr, out=out)
        torch.cuda.synchronize()
        _same(e_sc, d_sc, "d_sc")
        _same(ebias, dbias[:C], "dbias")
        assert bool(e_sc[..., :C].float().ne(0).any()) and not bool(e_sc[..., C:].float().ne(0).any())


# ---------------------------------------------------------------------------------------------------------------------
# 3. the training step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,C", [("COLOR", 2), ("COLOR", 10), ("COLOR", 22), ("RGBD", 10)])
def test_training_step_gradients(cuda, fmt, C):
    """B = 2, 64 x 96: every parameter's gradient against torch autograd of the segmentation graph, 16-bit-rounded and pure fp32,
    within train_ref.limits of the same layer names; then one step, and export_params() loads into the inference network."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.train import Trainer
    (data, gt, *_), _, depth = make_inputs(cuda, B=2, H=64, W=96, C=C)
    # at C = 2 the 0.02-scaled `score` starts confident (loss_cls 0.3): the small gradient that is left cancels down the trunk and
    # shows the bf16 rounding of the propagated gradient amplified; near-uniform logits keep every labelled pixel's term
    net = make_seg_net(cuda, fmt=fmt, C=C, score_scale=0.002 if C == 2 else 0.02)
    tr = Trainer(net, lr=0.01)
    assert not tr.pose_reg and tr.seg
    kw = dict(depth=depth) if fmt == "RGBD" else {}
    A = tr.forward(data, gt, **kw)
    assert "vtx_out" not in A and A["lowres"].shape == (2, 8, 12, C)
    grads = tr.backward(A, gt)
    torch.cuda.synchronize()
    assert set(grads) == set(tr.master)
    blob = torch.from_numpy(depth_blob_np(depth.cpu().numpy())).to(cuda) if fmt == "RGBD" else None
    P, loss16 = seg_reference_grads(net, data, gt, True, blob)
    Pf, loss32 = seg_reference_grads(net, data, gt, False, blob)
    got = float(A["cls_out"][0])
    print(f"loss_cls {got:.6f}  16-bit-rounded graph {loss16:.6f}  fp32 graph {loss32:.6f}")
    assert abs(got - loss16) < 2e-3 * abs(loss16) and abs(got - loss32) < 1e-2 * abs(loss32)
    compare_grads(tr, grads, P, Pf, sorted(grads))
    out = tr.step(data, gt, **kw)
    torch.cuda.synchronize()
    assert set(out) == {"loss_cls", "loss", "grads"} and torch.equal(out["loss"], out["loss_cls"])
    tr.export_params()
    inf = vgg16_convs(input_format=fmt, num_classes=C, device=cuda, vertex_reg_2d=False, vertex_reg_3d=False)
    inf.load({k: v.cpu() for k, v in net.params.items()})
    assert set(inf.params) == set(tr.layout[n][0] for n in tr.layout)
    for name in tr.master:
        tf = tr.layout[name][0]
        assert torch.equal(inf.params[tf], tr.to_tf(name, tr.master[name])), name
    L = inf.forward(data, None, None, want_prob=True, **kw)
    assert L["prob_normalized"].shape == (2, 64, 96, C)


# ---------------------------------------------------------------------------------------------------------------------
# 4. inference at batch 32
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["COLOR", "RGBD"])
def test_inference_graph_shards_and_evaluation(cuda, fmt):
    """Batch 32, 480 x 640, C = 10: GraphedForward's replay equals the eager pass; two image shards give the whole batch's label maps;
    Evaluator(num_classes=10).add_labels scores the output."""
    from posecnn_b200.evaluate import Evaluator
    from posecnn_b200.networks.vgg16_convs import GraphedForward
    B, H, W, C = 32, 480, 640, 10
    (data, gt, _, meta, ext, _, _, _), _, depth = make_inputs(cuda, B=B, H=H, W=W, C=C)
    seg = make_seg_net(cuda, fmt=fmt, C=C, is_train=False)
    kw = dict(depth=depth) if fmt == "RGBD" else {}
    seg.calibrate_background(data, meta, ext, **kw)
    eager = {k: v.clone() for k, v in seg.forward(data, meta, ext, want_prob=True, **kw).items()}
    g = GraphedForward(seg, data, meta, ext, want_prob=True, **kw)
    L = g(data, meta)
    torch.cuda.synchronize()
    for k in ("label_2d", "prob_normalized"):
        _same(L[k], eager[k], k)
    frac = float((eager["label_2d"] == 0).float().mean())
    print(f"{fmt}: background fraction {frac:.3f}")
    assert 0.5 < frac < 0.95
    parts = []
    for o in (0, B // 2):
        kws = dict(depth=depth[o:o + B // 2]) if fmt == "RGBD" else {}
        parts.append(seg.forward(data[o:o + B // 2], meta[o:o + B // 2], ext, batch_global=B, batch_offset=o, **kws)["label_2d"])
    _same(torch.cat(parts), eager["label_2d"], "label_2d of two shards")
    ev = Evaluator(num_classes=C, points=np.zeros((C, 1, 3)), extents=np.ones((C, 3)), symmetric=np.zeros(C), device=cuda)
    ev.add_labels(gt, eager["label_2d"])
    torch.cuda.synchronize()
    assert int(ev.hist.sum()) == int((gt >= 0).sum())


# ---------------------------------------------------------------------------------------------------------------------
# 5. two ranks
# ---------------------------------------------------------------------------------------------------------------------
SEG_WORKER = r'''
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
from posecnn_b200 import parallel
from posecnn_b200.train import Trainer
from tests.seg_ref import make_seg_net
from tests.train_ref import make_inputs
FMT = %(fmt)r
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
B, C = 4, 10
(data, gt, *_), _, dm = make_inputs(dev, B=B, C=C)
o, n = parallel.shard_range(B, rank, world)
whole, shard = (dict(depth=dm), dict(depth=dm[o:o + n])) if FMT == "RGBD" else ({}, {})
single = Trainer(make_seg_net(dev, fmt=FMT, C=C), lr=0.01)
ref = single.step(data, gt, **whole)
tr = Trainer(make_seg_net(dev, fmt=FMT, C=C), lr=0.01, world=world)
out = tr.step(data[o:o + n], gt[o:o + n], batch_global=B, batch_offset=o, **shard)
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
tot = out["loss_cls"].clone()
dist.all_reduce(tot)
assert torch.allclose(tot, ref["loss_cls"], rtol=1e-4, atol=1e-6), (tot, ref["loss_cls"])
dist.barrier()
dist.destroy_process_group()
print("SEG_RANK_OK", rank, worst)
'''


@pytest.mark.parametrize("fmt", ["COLOR", "RGBD"])
def test_two_rank_step_matches_one_rank(tmp_path, fmt):
    from tests.train_ref import ROOT
    run_two_ranks(tmp_path, SEG_WORKER % dict(root=ROOT, fmt=fmt), marker="SEG_RANK_OK")
