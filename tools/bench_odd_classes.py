"""Odd class counts: what the one-channel-per-thread forms of the up-sampling heads cost, C = 9 against its even neighbours C = 8
and C = 10, in one process on one GPU, arms alternating (C = 8, 9, 10 in turn, --runs times).

Inputs: a seeded synthetic 640x480 scene with C classes per arm (synth.make_scene, as bench.py --workload train forms its 22-class
scene), random low-resolution head tensors for the kernel arms.  Reported, median of the runs with every run listed:
  up8_heads       ms per launch of pcnn_up8_heads at batch --infer-batch (32): full mode (label, vertex_pred, prob, score) and the
                  pipeline's label-only mode (k_up8_label)
  up8_bwd         ms per launch of pcnn_up8_heads_bwd alone at batch --batch (64)
  infer           ms per forward of the inference network as one CUDA graph (GraphedForward, dense_vertex=False) at batch 32
  train           ms per step of the training step (pose_reg False: linemod_color_2d.yml) at batch --batch, CUDA events
The card name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/bench_odd_classes.py [--batch 64] [--infer-batch 32] [--steps 10] [--warmup 3] [--runs 3]
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
from bench_single_class import timed, timed_steps                  # noqa: E402
from bench_train_rgbd import H, W, gpu_info                        # noqa: E402
from posecnn_b200 import heads, synth                              # noqa: E402
from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs   # noqa: E402
from posecnn_b200.train import Trainer                             # noqa: E402

CLASSES = (8, 9, 10)


def make_inputs(dev, B, C):
    """The training batch of a C-class scene (8 distinct images repeated over the batch)."""
    nu = min(B, 8)
    sc = synth.make_scene(batch=nu, height=H, width=W, num_classes=C, seed=4234, other_channel_noise=False)
    reps = -(-B // nu)
    label = np.concatenate([sc["label"]] * reps, 0)[:B]
    centers = np.zeros((nu, C, 3), np.float32)
    for (b, cls, cx, cy, z) in sc["centers"]:
        centers[b, cls] = (cx, cy, z)
    centers = np.concatenate([centers] * reps, 0)[:B]
    gts = []
    for r in range(reps):
        g = sc["gt"].copy(); g[:, 0] += r * nu; gts.append(g)
    gt = np.concatenate(gts, 0); gt = gt[gt[:, 0] < B]
    rgb, _ = synth.make_images(B, H, W, seed=21)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return (T(rgb), T(label), T(centers), T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)), T(synth.extents_for(C)), T(gt),
            T(synth.make_model_points(C, 2620)), torch.zeros(C, device=dev))


def make_trainer(dev, C):
    net = vgg16_convs(num_classes=C, device=dev, is_train=True, fold_vertex_head=False, pose_reg=False).init_random(seed=0)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02
    net.prepare()
    return Trainer(net, lr=1e-4, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0)


def heads_arms(dev, B, C):
    """pcnn_up8_heads on a random low-resolution tensor: the full call and the label-only call."""
    h, w = H // 8, W // 8
    g = torch.Generator().manual_seed(C)
    lowres = (torch.randn(B, h, w, 4 * C, generator=g) * 0.7).to(dev)
    bs, bv = (torch.randn(C, generator=g) * 0.1).to(dev), (torch.randn(3 * C, generator=g) * 0.1).to(dev)
    out = heads.up8_heads(lowres, bs, bv, vertex=True, prob=True, score=True)

    def full():
        heads.up8_heads(lowres, bs, bv, out=out)

    def label_only():
        heads.up8_heads(lowres, bs, bv, out=(out[0], None, None, None))
    return full, label_only


def bwd_arm(dev, B, C, gt):
    """pcnn_up8_heads_bwd on the heads of a random low-resolution tensor and the scene's labels."""
    h, w = H // 8, W // 8
    g = torch.Generator().manual_seed(100 + C)
    lowres = (torch.randn(B, h, w, 4 * C, generator=g) * 0.7).to(dev)
    bs, bv = (torch.randn(C, generator=g) * 0.1).to(dev), (torch.randn(3 * C, generator=g) * 0.1).to(dev)
    _, _, prob, score = heads.up8_heads(lowres, bs, bv, prob=True, score=True)
    centers = torch.zeros((B, C, 3), device=dev)
    centers[:, 1:, 0], centers[:, 1:, 1], centers[:, 1:, 2] = W / 2, H / 2, 1.0
    cls_out, vtx_out = torch.tensor([0.5, 1e5], device=dev), torch.tensor([0.5, 1e5], device=dev)
    out = heads.up8_heads_bwd(prob, score, gt, cls_out, 1.0, 0.7, lowres, bv, centers, vtx_out, 1.0, 10.0, 1.0)

    def run():
        heads.up8_heads_bwd(prob, score, gt, cls_out, 1.0, 0.7, lowres, bv, centers, vtx_out, 1.0, 10.0, 1.0, out=out)
    return run


def alternate(arms, runs, fn):
    res = {k: [] for k in arms}
    for _ in range(runs):
        for k, arm in arms.items():
            res[k].append(fn(arm))
    return {k: dict(ms=statistics.median(v), ms_runs=v) for k, v in res.items()}


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
    out = dict(metric="odd class count (C = 9) against C = 8 and 10", batch=B, infer_batch=Bi, image=f"{W}x{H}", steps=a.steps,
               warmup=a.warmup, runs=a.runs, gpu=info["name"], power_limit=info["power_limit"])
    inputs = {C: make_inputs(dev, B, C) for C in CLASSES}
    # ---- the kernels alone
    heads = {C: heads_arms(dev, Bi, C) for C in CLASSES}
    for k, r in alternate({C: f for C, (f, _) in heads.items()}, a.runs, lambda fn: timed(fn, 20)).items():
        out[f"up8_heads_full_c{k}"] = r
    for k, r in alternate({C: f for C, (_, f) in heads.items()}, a.runs, lambda fn: timed(fn, 20)).items():
        out[f"up8_heads_label_only_c{k}"] = r
    del heads
    bwd = {C: bwd_arm(dev, B, C, inputs[C][1]) for C in CLASSES}
    for k, r in alternate(bwd, a.runs, lambda fn: timed(fn, 20)).items():
        out[f"up8_bwd_c{k}"] = r
    del bwd
    torch.cuda.empty_cache()
    # ---- inference: one CUDA graph per class count
    graphs = {}
    for C in CLASSES:
        net = vgg16_convs(num_classes=C, device=dev).init_random(seed=0)
        data, meta, ext = inputs[C][0][:Bi], inputs[C][3][:Bi], inputs[C][4]
        net.calibrate_background(data, meta, ext, 0.75)
        graphs[C] = (GraphedForward(net, data, meta, ext, dense_vertex=False), data)
    for k, r in alternate(graphs, a.runs, lambda gd: timed(lambda: gd[0](gd[1]), 20)).items():
        out[f"infer_c{k}_b{Bi}"] = dict(r, frames_per_s=Bi / (r["ms"] * 1e-3))
    del graphs
    torch.cuda.empty_cache()
    # ---- the training step (pose_reg False)
    trainers = {C: (make_trainer(dev, C), inputs[C]) for C in CLASSES}
    for k, r in alternate(trainers, a.runs, lambda ta: timed_steps(ta[0], ta[1], a.steps, a.warmup)[0]).items():
        out[f"train_c{k}_b{B}"] = dict(r, frames_per_s=B / (r["ms"] * 1e-3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
