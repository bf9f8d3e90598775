"""Shared harness of the training-step tests: the seeded test problem, torch fp32 autograd of the training graph (colour, RGB-D
and the domain branch) restated on oracle/ref_network.py with the reference's losses (lib/fcn/train.py:455-465, 508-513,
564-573; Averagedistance formula average_distance_loss_op_gpu.cu.cc:34-252), the gradient comparison with its stated limits,
and the two-rank worker."""
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

MEANS = (102.9801, 115.9465, 122.7717)
LAMBDA = 0.01
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_l2(a, b):
    return ((a - b).pow(2).sum() / b.pow(2).sum().clamp(min=1e-30)).sqrt().item()


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def depth_blob_np(depth_mm):
    """The depth blob of lib/fcn/test.py:70-76 in numpy float32: clip(d / 2000, 0, 1) * 255 tiled x3 - PIXEL_MEANS -> [B,H,W,3]."""
    d = np.asarray(depth_mm, np.float32)
    g = np.clip(d / np.float32(2000.0), np.float32(0.0), np.float32(1.0)) * np.float32(255.0)
    return (g[..., None] - np.asarray(MEANS, np.float32)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# the test problem
# ---------------------------------------------------------------------------------------------------------------------
def make_net(cuda, fmt="COLOR", adaptation=False, is_train=True, C=6, seed=0):
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(input_format=fmt, num_classes=C, device=cuda, is_train=is_train, fold_vertex_head=False,
                      adaptation=adaptation).init_random(seed=seed, bias_std=0.02)
    # bring the three output layers to O(1) logits / pre-activations so that neither the softmax nor the tanh saturates
    net.params["score/weights"] *= 0.02
    net.params["vertex_pred/weights"] *= 0.02
    net.params["fc8/weights"] *= 0.01
    if adaptation:      # O(1) domain logits: a saturated softmax leaves only fp32 cancellation noise in the reference's gradient
        net.params["domain_score/weights"] *= 0.05
    net.prepare()
    return net


def make_inputs(cuda, B=2, H=64, W=96, C=6):
    """(labelled, adapt, depth): the labelled batch (data, gt_label_2d, centers, meta_data, extents, gt_poses, points, symmetry);
    its adapt form (labels -1 everywhere, no gt poses, no centres); a raw depth image in millimetres (synth depth x 1000, as
    bench.py --workload rgbd feeds it)."""
    rgb, depth = synth.make_images(B, H, W, seed=3)
    sc = synth.make_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=3, seed=11, min_pixels=200)
    centers = np.zeros((B, C, 3), np.float32)
    for (b, cls, cx, cy, z) in sc["centers"]:
        centers[b, cls] = (cx, cy, z)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    labelled = (T(rgb), T(sc["label"]), T(centers), T(sc["meta"].reshape(B, 48)), T(sc["extents"]), T(sc["gt"]),
                T(synth.make_model_points(C, 300)), torch.zeros(C, device=cuda))
    adapt = (labelled[0], torch.full_like(labelled[1], -1), torch.zeros_like(labelled[2]), labelled[3], labelled[4],
             torch.zeros((0, 13), device=cuda), labelled[6], labelled[7])
    return labelled, adapt, T((depth * 1000.0).astype(np.float32))


def synthetic_pose_targets(A, pts, sym, margin):
    """Quaternion targets on the ROI rows' own classes (the Hough targets depend on gt boxes overlapping the ROIs): replaces the
    forward's pose targets, loss and Averagedistance gradient in A.  Returns (targets, weights)."""
    from posecnn_b200.average_distance_loss import average_distance_loss_op
    rows, D = A["poses_tanh"].shape
    g = torch.Generator().manual_seed(5)
    tw, wt = torch.zeros(rows, D), torch.zeros(rows, D)
    for r in range(rows):
        c = int(A["rois"][r, 1].item())
        q = torch.randn(4, generator=g); q = q / q.norm()
        tw[r, 4 * c:4 * c + 4] = q; wt[r, 4 * c:4 * c + 4] = 1.0
    tw, wt = tw.to(pts.device), wt.to(pts.device)
    mul = A["poses_tanh"] * wt
    pred = (mul / mul.pow(2).sum(1, keepdim=True).clamp(min=1e-12).sqrt()).contiguous()
    A["loss_pose_raw"], A["pose_diff"] = average_distance_loss_op.average_distance_loss(pred, tw, wt, pts, sym, margin)
    A["poses_weight"], A["poses_target"] = wt, tw
    return tw, wt


def grads_of(tr, args, **kw):
    """The gradients of one forward + backward of Trainer tr (no update), cloned."""
    A = tr.forward(*args, **kw)
    g = tr.backward(A, args[1], args[2])
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in g.items()}


# ---------------------------------------------------------------------------------------------------------------------
# the autograd reference
# ---------------------------------------------------------------------------------------------------------------------
def quat_rot(q):
    s, u, v, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]          # un-normalised formula, .cu.cc:63-71
    return torch.stack([s * s + u * u - v * v - w * w, 2 * (u * v - s * w), 2 * (u * w + s * v),
                        2 * (u * v + s * w), s * s - u * u + v * v - w * w, 2 * (v * w - s * u),
                        2 * (u * w - s * v), 2 * (v * w + s * u), s * s - u * u - v * v + w * w], -1).reshape(*q.shape[:-1], 3, 3)


def ad_loss_torch(pred, target, weight, points, margin):
    """Averagedistance for non-symmetric classes, differentiable in pred."""
    N, D = pred.shape
    C = D // 4
    loss = pred.new_zeros(())
    P = points.shape[1]
    for n in range(N):
        cls = next((i for i in range(C) if weight[n, 4 * i] > 0), -1)
        if cls < 0:
            continue
        Ru, Rg = quat_rot(pred[n, 4 * cls:4 * cls + 4]), quat_rot(target[n, 4 * cls:4 * cls + 4])
        a, b = points[cls] @ Ru.t(), points[cls] @ Rg.t()
        d = (a - b).pow(2).sum(1)
        loss = loss + torch.where(d < margin, torch.zeros_like(d), d - margin).sum() / (2.0 * N * P)
    return loss


def _ste(y, dtype):
    """Round to a 16-bit format in the forward pass, identity in the backward pass (what storing an activation in bf16 / fp16 does)."""
    return y + (y.to(dtype).float() - y).detach()


class GradReverse(torch.autograd.Function):
    """gradient_reversal_op_gpu.cu.cc: identity forward, -lambda * grad backward."""
    @staticmethod
    def forward(ctx, x, lam):
        ctx.lam = lam
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return -ctx.lam * g, None


def reference_grads(net, A, inputs, targets, weights, sim16, vertex_w=1.0, w_inside=10.0, margin=0.01, depth_blob=None,
                    adapt_weight=None, domain_only=False, lam=LAMBDA):
    """torch fp32 autograd of the same losses on the same inputs (the labelled-batch tuple of make_inputs); ROI pooling gathers at
    OUR arg-max positions, label_domain is Hough's.  Returns the parameters (with .grad) and a dict of the losses and outputs.
    sim16=False: the reference graph in the reference's op order, pure fp32 (oracle/ref_network.py).
    sim16=True:  the same mathematics in THIS implementation's op order (1x1 before the x8 up-sampling) with every stored activation
    rounded to bf16 (trunk, heads) / fp16 (pose head) where our kernels round it — isolates kernel errors from precision effects.
    depth_blob [B,H,W,3]: the RGB-D graph, its depth trunk on that blob; score_conv4 / 5 read the concat [colour | depth].
    adapt_weight: adds pool_score -> GradReverse(lam) -> fc9 -> ReLU -> domain_score -> ReLU -> cross entropy (the domain branch);
    domain_only: loss = loss_domain alone."""
    data, gt, centers, points = inputs[0], inputs[1], inputs[2], inputs[6]
    P = {k: v.detach().clone().requires_grad_(True) for k, v in net.params.items()}
    C = net.num_classes
    bf, hf = torch.bfloat16, torch.float16
    r16 = (lambda y: _ste(y, bf)) if sim16 else (lambda y: y)
    rh = (lambda y: _ste(y, hf)) if sim16 else (lambda y: y)
    W = (lambda w: _ste(w, bf)) if sim16 else (lambda w: w)          # bf16 tensor-core copies of the weights
    Wh = (lambda w: _ste(w, hf)) if sim16 else (lambda w: w)

    def trunk(x, sfx):
        x = r16(x)
        feats = {}
        for item in R.VGG_CFG:
            if isinstance(item, str):
                x = F.max_pool2d(x, 2)
            else:
                x = r16(R.conv(x, W(P[f"{item[0]}{sfx}/weights"]), P[f"{item[0]}{sfx}/biases"]))
                feats[item[0]] = x
        return feats
    f = trunk((data.float() - torch.tensor(MEANS, device=data.device)).permute(0, 3, 1, 2), "")
    c4, c5 = f["conv4_3"], f["conv5_3"]
    h4, h5 = c4, c5
    if depth_blob is not None:
        fp = trunk(depth_blob.permute(0, 3, 1, 2), "_p")
        h4, h5 = torch.cat([c4, fp["conv4_3"]], 1), torch.cat([c5, fp["conv5_3"]], 1)    # concat_conv4 / 5, colour first
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
    ps.retain_grad()
    h6 = rh(torch.relu(ps @ Wh(P["fc6/weights"]) + P["fc6/biases"]))
    h7 = rh(torch.relu(h6 @ Wh(P["fc7/weights"]) + P["fc7/biases"]))
    th = torch.tanh(h7 @ Wh(P["fc8/weights"]) + P["fc8/biases"])
    mul = th * weights
    pred = mul / mul.pow(2).sum(1, keepdim=True).clamp(min=1e-12).sqrt()
    loss_pose = ad_loss_torch(pred, targets, weights, points, margin)
    loss = loss_cls + vertex_w * loss_vertex + loss_pose
    out = dict(loss_cls=loss_cls.item(), loss_vertex=(vertex_w * loss_vertex).item(), loss_pose=loss_pose.item(), score=score.detach(),
               vertex=vertex.detach(), tanh=th.detach())
    if adapt_weight is not None:
        h9 = rh(torch.relu(GradReverse.apply(ps, lam) @ Wh(P["fc9/weights"]) + P["fc9/biases"]))
        z = torch.relu(h9 @ P["domain_score/weights"] + P["domain_score/biases"])
        loss_domain = adapt_weight * F.cross_entropy(z, A["label_domain"].long())
        loss = loss_domain if domain_only else loss + loss_domain
        out.update(loss_domain=loss_domain.item(), domain_score=z.detach())
    loss.backward()
    out.update(dpool=ps.grad.detach())
    return P, out


# ---------------------------------------------------------------------------------------------------------------------
# the comparison
# ---------------------------------------------------------------------------------------------------------------------
def limits(name):
    """(16-bit-rounded, pure fp32) relative-L2 limits of a Trainer gradient.  Kernel correctness (16-bit-rounded graph): same masks,
    same rounding points -> only the 16-bit rounding of the PROPAGATED gradients is left (the reference keeps them in fp32); weight /
    bias gradients are cancellation-heavy sums, so that rounding noise shows amplified: measured 0.1-0.7e-2 on the heads, 2e-2 ->
    4e-2 down the trunk, 7e-2 / 1.2e-1 on the conv1_2 / conv1_1 weights.  Pose head: d loss / d poses_tanh after l2_normalize is
    what is left when the radial component of Averagedistance's gradient is removed — a cancellation residual, so the 1e-3 relative
    differences of an fp16 forward show up as 1e-2 .. 1e-1 in fc6 / fc7 / fc8 gradients (|ref| 1e-6 .. 1e-2); the GEMMs themselves
    are checked to 2e-3 / 1e-4 in tests/test_backward_gpu.py.  Pure fp32 graph: ReLU / max-pool masks of a bf16 forward differ from
    the fp32 ones for near-tie activations, which compounds with depth; weight gradients of the first block are cancellation-heavy.
    A `_p` layer gets its colour counterpart's limits, fc9 fc6's, domain_score the heads'."""
    base = name.replace("_p/", "/").replace("fc9/", "fc6/")
    layer = base.split("/")[0]
    lim16 = 0.2 if base == "conv1_1/w" else (0.15 if layer in ("conv1_1", "conv1_2", "fc6", "fc7", "fc8") else 6e-2)
    lim32 = 0.3 if layer in ("conv1_1", "conv1_2") else (0.15 if layer in ("fc6", "fc7", "fc8") else 0.1)
    return lim16, lim32


def limits_adapt(name):
    """The adapt batch's trunk gradients have one sparse source (the reversed domain gradient scattered by RoiPool at the ROI
    maxima), and their weight gradients cancel more than the colour step's: the bf16 rounding of the propagated gradient shows
    amplified further down.  Measured on this problem (16-bit-rounded / pure fp32 graph): 0.04-0.06 / 0.05-0.07 for conv5_x,
    0.05-0.08 / 0.06-0.10 for conv4_x, 0.09-0.13 / 0.11-0.16 for conv3_x and 0.13-0.17 / 0.19-0.28 for conv1_x-conv2_x."""
    block = name.split("/")[0][:5]
    if block in ("conv5", "conv4"):
        return 0.12, 0.15
    return (0.2, 0.25) if block == "conv3" else (0.3, 0.4)


def compare_grads(tr, grads, P, Pf, names, limits=limits):
    """Every gradient in `names` against the 16-bit-rounded (P) and the pure fp32 (Pf) autograd graph, in TF layout; prints each
    error, then asserts the limits."""
    errs = {}
    for name in names:
        layer, kind = name.split("/")
        key = f"{layer}/{'weights' if kind == 'w' else 'biases'}"
        got = tr.to_tf(name, grads[name])
        assert got.shape == P[key].grad.shape, name
        e16, e32 = rel_l2(got, P[key].grad), rel_l2(got, Pf[key].grad)
        print(f"grad {name:26s} rel-L2 vs 16-bit-rounded graph {e16:.3e}   vs pure fp32 graph {e32:.3e}   |ref| {P[key].grad.norm().item():.3e}")
        errs[name] = (e16, e32)
    for name, (e16, e32) in errs.items():
        lim16, lim32 = limits(name)
        assert e16 < lim16, (name, e16, lim16)
        assert e32 < lim32, (name, e32, lim32)


# ---------------------------------------------------------------------------------------------------------------------
# two ranks
# ---------------------------------------------------------------------------------------------------------------------
TRAIN_WORKER = r'''
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
from posecnn_b200 import parallel
from posecnn_b200.networks.vgg16_convs import vgg16_convs
from posecnn_b200.train import Trainer
from tests.train_ref import make_inputs
FMT, ADAPT = %(fmt)r, %(adapt)r
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
B, C = 4, 6
def trainer(world):
    net = vgg16_convs(input_format=FMT, num_classes=C, device=dev, is_train=True, fold_vertex_head=False,
                      adaptation=ADAPT).init_random(seed=0, bias_std=0.02)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02; net.params["fc8/weights"] *= 0.01
    net.prepare()
    return Trainer(net, lr=0.01, world=world, **(dict(adapt_weight=1.0) if ADAPT else {}))
(data, gt, cen, meta, ext, gtp, pts, sym), _, dm = make_inputs(dev, B=B, C=C)
if ADAPT:
    gtp = gtp[gtp[:, 0] < 2]                   # gt poses on the first shard's images only: rank 1 has none of its own
o, n = parallel.shard_range(B, rank, world)
whole, shard = (dict(depth=dm), dict(depth=dm[o:o + n])) if FMT == "RGBD" else ({}, {})
single = trainer(1)
ref = single.step(data, gt, cen, meta, ext, gtp, pts, sym, **whole)
tr = trainer(world)
out = tr.step(data[o:o + n], gt[o:o + n], cen[o:o + n], meta[o:o + n], ext, gtp, pts, sym, batch_global=B, batch_offset=o, **shard)
torch.cuda.synchronize()
if ADAPT:
    assert not bool(out["label_domain"].any())     # decided by the whole batch's gt count, on every rank
assert set(out["grads"]) == set(ref["grads"]) == set(tr.master)
worst = 0.0
for name, g in out["grads"].items():
    w = ref["grads"][name]
    e = ((g - w).norm() / w.norm().clamp(min=1e-20)).item()
    worst = max(worst, e)
    assert e < 2e-3, (name, e)
for name in tr.master:
    assert torch.allclose(tr.master[name], single.master[name], rtol=1e-4, atol=1e-6), name
losses = ["loss_cls", "loss_vertex", "loss_pose"] + (["loss_domain"] if ADAPT else [])
tot = torch.stack([out[k][0] for k in losses])
dist.all_reduce(tot)
want = torch.stack([ref[k][0] for k in losses])
assert torch.allclose(tot, want, rtol=1e-4, atol=1e-6), (tot, want)
dist.barrier()
dist.destroy_process_group()
print("TRAIN_RANK_OK", rank, worst)
'''


def train_worker(fmt="COLOR", adaptation=False):
    """The two-rank training worker: one SGD step on image shards over 2 ranks against the step on the whole batch on one GPU."""
    return TRAIN_WORKER % dict(root=ROOT, fmt=fmt, adapt=adaptation)


def run_two_ranks(tmp_path, script, marker="TRAIN_RANK_OK", timeout=900):
    """Run `script` on 2 ranks (torch.distributed.run, NCCL); both must print `marker`.  Skips on a machine with fewer GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    path = tmp_path / "worker.py"
    path.write_text(script)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), str(path)], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0 and out.stdout.count(marker) == 2, (out.stdout[-2000:], out.stderr[-3000:])
