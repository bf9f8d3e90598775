"""Segmentation network (vgg16_convs with vertex_reg_2d = vertex_reg_3d = False: rgbd_scene_single_*.yml, shapenet_*_single_*.yml,
lov_single_color_*.yml) against the 2-D vertex network at the same class count, in one process on one GPU, the two arms alternating
(--runs times).

Inputs: a seeded synthetic 640x480 scene with C classes (synth.make_scene, as bench.py --workload train forms its scene) and its
depth image in millimetres for the RGB-D arms.  Reported, median of the runs with every run listed:
  infer     ms per forward as one CUDA graph (GraphedForward) at batch --infer-batch (32): the segmentation network against the 2-D
            network in the pipeline mode (dense_vertex=False), C = 10 and 22, colour and RGB-D
  train     ms per training step at batch --batch (64): the segmentation step (loss_cls) against the 2-D pose_reg=False step
            (loss_cls + loss_vertex), C = 10 and 22 colour and C = 10 RGB-D, CUDA events
  up8_bwd   ms per launch of the loss-gradient adjoint alone at batch --batch: target mode "none" (pcnn_up8_scores_bwd) against the
            2-D mode (pcnn_up8_heads_bwd), on the heads of a random low-resolution tensor and the scene's labels
The card name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/bench_segmentation.py [--batch 64] [--infer-batch 32] [--steps 10] [--warmup 3] [--runs 3]
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
from bench_odd_classes import make_inputs                          # noqa: E402
from bench_single_class import timed                               # noqa: E402
from bench_train_rgbd import H, W, gpu_info                        # noqa: E402
from posecnn_b200 import heads, synth                              # noqa: E402
from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs   # noqa: E402
from posecnn_b200.train import Trainer                             # noqa: E402


def alternate(arms, runs, fn):
    res = {k: [] for k in arms}
    for _ in range(runs):
        for k, arm in arms.items():
            res[k].append(fn(arm))
    return {k: dict(ms=statistics.median(v), ms_runs=v) for k, v in res.items()}


def make_net(dev, fmt, C, seg, **kw):
    net = vgg16_convs(input_format=fmt, num_classes=C, device=dev, vertex_reg_2d=not seg, vertex_reg_3d=False, **kw).init_random(seed=0)
    net.params["score/weights"] *= 0.02
    if not seg:
        net.params["vertex_pred/weights"] *= 0.02
    net.prepare()
    return net


def bwd_arms(dev, B, C, gt):
    """The two adjoint launches on the heads of a random low-resolution tensor and the scene's labels."""
    h, w = H // 8, W // 8
    g = torch.Generator().manual_seed(C)
    lowres = (torch.randn((B, h, w, 4 * C), generator=g) * 2.0).to(dev)
    bs, bv = torch.zeros(C, device=dev), torch.zeros(3 * C, device=dev)
    _, _, prob, score = heads.up8_heads(lowres, bs, bv, prob=True, score=True)
    centers = torch.zeros((B, C, 3), device=dev)
    centers[..., 0], centers[..., 1], centers[..., 2] = W / 2, H / 2, 1.0
    cls_out, vtx_out = torch.tensor([1.0, float(B * H * W)], device=dev), torch.tensor([1.0, 1000.0], device=dev)
    out2 = heads.up8_heads_bwd(prob, score, gt, cls_out, 1.0, 0.7, lowres, bv, centers, vtx_out, 1.0, 10.0, 1.0)
    out0 = heads.up8_scores_bwd(prob, score, gt, cls_out, 1.0, 0.7)
    return {"none": lambda: heads.up8_scores_bwd(prob, score, gt, cls_out, 1.0, 0.7, out=out0),
            "2d": lambda: heads.up8_heads_bwd(prob, score, gt, cls_out, 1.0, 0.7, lowres, bv, centers, vtx_out, 1.0, 10.0, 1.0, out=out2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--infer-batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info()
    B, Bi = a.batch, a.infer_batch
    out = dict(metric="segmentation network (no vertex head) against the 2-D vertex network", batch=B, infer_batch=Bi, image=f"{W}x{H}",
               steps=a.steps, warmup=a.warmup, runs=a.runs, gpu=info["name"], power_limit=info["power_limit"])
    _, depth = synth.make_images(B, H, W, seed=21)
    depth = torch.from_numpy((depth * 1000.0).astype(np.float32)).to(dev)
    for C in (10, 22):
        inputs = make_inputs(dev, B, C)
        # ---- the adjoint alone
        for k, r in alternate(bwd_arms(dev, B, C, inputs[1]), a.runs, lambda fn: timed(fn, 20)).items():
            out[f"up8_bwd_{k}_c{C}_b{B}"] = r
        # ---- inference graphs
        for fmt in ("COLOR", "RGBD"):
            data, meta, ext = inputs[0][:Bi], inputs[3][:Bi], inputs[4]
            kw = dict(depth=depth[:Bi]) if fmt == "RGBD" else {}
            graphs = {}
            for arm, seg in (("seg", True), ("2d", False)):
                net = make_net(dev, fmt, C, seg)
                net.calibrate_background(data, meta, ext, 0.75, **kw)
                graphs[arm] = (GraphedForward(net, data, meta, ext, **(kw if seg else dict(kw, dense_vertex=False))), data)
            for k, r in alternate(graphs, a.runs, lambda gd: timed(lambda: gd[0](gd[1]), 20)).items():
                out[f"infer_{k}_{fmt.lower()}_c{C}_b{Bi}"] = dict(r, frames_per_s=Bi / (r["ms"] * 1e-3))
            del graphs
            torch.cuda.empty_cache()
        # ---- the training step
        for fmt in ("COLOR", "RGBD") if C == 10 else ("COLOR",):
            kw = dict(depth=depth) if fmt == "RGBD" else {}
            trainers = {arm: Trainer(make_net(dev, fmt, C, seg, is_train=True, fold_vertex_head=False, pose_reg=False), lr=1e-4)
                        for arm, seg in (("seg", True), ("2d", False))}
            step = lambda tr: timed(lambda: tr.step(*inputs, **kw), a.steps, a.warmup)
            for k, r in alternate(trainers, a.runs, step).items():
                out[f"train_{k}_{fmt.lower()}_c{C}_b{B}"] = dict(r, frames_per_s=B / (r["ms"] * 1e-3))
            del trainers
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
