"""Single-object (num_classes = 2) models against the 22-class model, in one process on one GPU, arms alternating.

Inputs: the seeded synthetic 640x480 scene of `bench.py --workload train` (tools/bench_train_rgbd.py make_inputs: 22 classes); the
two-class arms see its single-class view (posecnn_b200.single_class) for the class with the most labelled pixels, as the
reference's loader forms it for a LINEMOD / per-object YCB model.  Reported:
  train   ms per step at --batch (64) of the C = 22 step, the C = 2 step (pose_reg True) and the C = 2 step without the pose head
          (pose_reg False, the linemod_{benchvise,camera,iron,lamp,phone}.yml models); --runs runs of --warmup + --steps steps
          each, the three arms in turn, CUDA events
  infer   ms per forward of the C = 2 inference network as one CUDA graph (GraphedForward, dense_vertex=False) at batch 32 and 1
  up8_bwd ms per launch of pcnn_up8_heads_bwd_ex alone (the loss-gradient up-sampling adjoint) at C = 2 and C = 22, batch --batch,
          60 x 80 low-resolution cells, the two class counts alternating
The card name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/bench_single_class.py [--batch 64] [--steps 10] [--warmup 3] [--runs 3]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_train_rgbd import H, W, gpu_info, make_inputs           # noqa: E402
from posecnn_b200._lib import check, lib, ptr, stream        # noqa: E402
from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs   # noqa: E402
from posecnn_b200.single_class import single_class_view           # noqa: E402
from posecnn_b200.train import Trainer                             # noqa: E402


def make_trainer(dev, C, pose_reg=True):
    net = vgg16_convs(num_classes=C, device=dev, is_train=True, fold_vertex_head=False, pose_reg=pose_reg).init_random(seed=0)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02; net.params["fc8/weights"] *= 0.01
    net.prepare()
    return Trainer(net, lr=1e-4, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0, margin=0.01)


def two_class_inputs(args):
    data, gt, centers, meta, ext, gtp, pts, sym = args
    counts = torch.bincount(gt.flatten().long().clamp(min=0), minlength=centers.shape[1])
    cls = int(counts[1:].argmax()) + 1
    v = single_class_view(cls, gt, centers, gtp, ext, pts, sym)
    return cls, (data, v["label"], v["centers"], meta, v["extents"], v["gt_poses"], v["points"], v["symmetry"])


def timed_steps(tr, args, steps, warmup):
    for _ in range(warmup):
        tr.step(*args)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = tr.step(*args)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, {k: float(v.item()) for k, v in out.items() if k.startswith("loss")}


def timed(fn, n, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def up8_problem(dev, B, C, gt):
    """Heads of a random low-resolution tensor (pcnn_up8_heads) with the scene's labels mapped into 0..C-1, and the launch."""
    h, w = H // 8, W // 8
    g = torch.Generator().manual_seed(C)
    lowres = (torch.randn(B, h, w, 4 * C, generator=g) * 0.7).to(dev)
    bs, bv = (torch.randn(C, generator=g) * 0.1).to(dev), (torch.randn(3 * C, generator=g) * 0.1).to(dev)
    label = torch.empty((B, H, W), dtype=torch.int32, device=dev)
    prob, score = torch.empty((B, H, W, C), device=dev), torch.empty((B, H, W, C), device=dev)
    check(lib().pcnn_up8_heads(ptr(lowres), ptr(bs), ptr(bv), B, h, w, C, ptr(label), ptr(None), ptr(prob), ptr(score), stream()))
    lab = (gt % C).contiguous() if C > 2 else (gt > 0).to(torch.int32)
    centers = torch.zeros((B, C, 3), device=dev)
    centers[:, 1:, 0], centers[:, 1:, 1], centers[:, 1:, 2] = W / 2, H / 2, 1.0
    cls_out, vtx_out = torch.tensor([0.5, 1e5], device=dev), torch.tensor([0.5, 1e5], device=dev)
    d_sc = torch.empty((B, h, w, 64), dtype=torch.bfloat16, device=dev)
    d_vt = torch.empty((B, h, w, 128), dtype=torch.bfloat16, device=dev)
    dbias = torch.empty((4 * C,), device=dev)
    ws = torch.empty(4 * B * ((w + 3) // 4) * ((h + 15) // 16) * 4 * C, dtype=torch.uint8, device=dev)

    def run():
        check(lib().pcnn_up8_heads_bwd_ex(ptr(prob), ptr(score), ptr(lab), ptr(cls_out), 1.0, 0.7, ptr(None), ptr(lowres), ptr(bv),
                                          ptr(centers), ptr(vtx_out), 1.0, 10.0, 1.0, B, h, w, C, 64, 128, ptr(d_sc), ptr(d_vt),
                                          ptr(dbias), ptr(ws), ws.numel(), stream()))
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info()
    B = a.batch
    args22, _ = make_inputs(dev, B)
    cls, args2 = two_class_inputs(args22)
    out = dict(metric="single-object (C = 2) models vs the 22-class model", batch=B, image=f"{W}x{H}", steps=a.steps, warmup=a.warmup,
               runs=a.runs, cls_index=cls, gpu=info["name"], power_limit=info["power_limit"])
    # ---- training step
    arms = {"train_c22": (make_trainer(dev, 22), args22), "train_c2": (make_trainer(dev, 2), args2),
            "train_c2_no_pose_reg": (make_trainer(dev, 2, pose_reg=False), args2)}
    res = {k: [] for k in arms}
    losses = {}
    for _ in range(a.runs):
        for k, (tr, args) in arms.items():
            ms, losses[k] = timed_steps(tr, args, a.steps, a.warmup)
            assert all(np.isfinite(v) for v in losses[k].values()), (k, losses[k])
            res[k].append(ms)
    for k in arms:
        out[k] = dict(ms_per_step=statistics.median(res[k]), ms_per_step_runs=res[k], frames_per_s=B / (statistics.median(res[k]) * 1e-3),
                      last_losses=losses[k])
    del arms
    torch.cuda.empty_cache()
    # ---- inference, one CUDA graph per batch size
    net = vgg16_convs(num_classes=2, device=dev).init_random(seed=0)
    data, meta, ext = args2[0], args2[3], args2[4]
    net.calibrate_background(data[:32], meta[:32], ext, 0.75)
    for nb in (32, 1):
        g = GraphedForward(net, data[:nb], meta[:nb], ext, dense_vertex=False)
        runs = [timed(lambda: g(data[:nb]), 20) for _ in range(a.runs)]
        out[f"infer_c2_b{nb}"] = dict(ms_per_forward=statistics.median(runs), ms_runs=runs, frames_per_s=nb / (statistics.median(runs) * 1e-3))
        del g
    del net
    torch.cuda.empty_cache()
    # ---- the up-sampling adjoint alone
    kern = {C: up8_problem(dev, B, C, args22[1]) for C in (2, 22)}
    kres = {C: [] for C in kern}
    for _ in range(a.runs):
        for C, fn in kern.items():
            kres[C].append(timed(fn, 20))
    for C in kern:
        out[f"up8_bwd_c{C}"] = dict(ms_per_launch=statistics.median(kres[C]), ms_runs=kres[C])
    out["ratio_train_c2_over_c22"] = out["train_c2"]["ms_per_step"] / out["train_c22"]["ms_per_step"]
    out["ratio_train_c2_no_pose_reg_over_c22"] = out["train_c2_no_pose_reg"]["ms_per_step"] / out["train_c22"]["ms_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
