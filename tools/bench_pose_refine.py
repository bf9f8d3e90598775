"""Cost of the depth pose refinement (csrc/pose_refine.cu) on one GPU; prints one JSON line.

  refine     batch 32 at 640 x 480, up to 4 ROIs per image on analytic depth scenes (synth.make_refine_scene, sigma = 1 mm),
             2620-point tables, 8 hypotheses x 8 iterations: ms per batch (histogram + refinement launch) and per ROI
  graphed    GraphedForward of vgg16_convs (C = 22, batch 32, 480 x 640) ms/step without and with refine_depth

    python tools/bench_pose_refine.py [--steps 20] [--warmup 3] [--batch 32]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from posecnn_b200 import synth  # noqa: E402
from posecnn_b200.pose_refine import refine_poses  # noqa: E402


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    B, H, W, C = args.batch, 480, 640, 22
    sc = synth.make_refine_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=4, seed=3, noise_m=0.001, min_pixels=400)
    rng = np.random.default_rng(0)
    rois, poses = [], []
    for row in sc["poses"]:
        qp, tp = synth.perturb_pose(row[2:6], row[6:9], rng)
        rois.append([row[0], row[1], 0, 0, 1, 1, 1.0])
        poses.append(np.r_[qp, tp])
    n = len(rois)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32) if np.asarray(a).dtype == np.float64 else a)).to(dev)
    lab, dep, meta = T(sc["label"]), T(sc["depth"]), T(sc["meta"])
    r, p, pts = T(np.array(rois)), T(np.array(poses)), T(sc["points"])
    num = torch.tensor([n], dtype=torch.int32, device=dev)
    ms_refine = time_ms(lambda: refine_poses(lab, dep, meta, r, p, pts, num_rows=num), args.steps, args.warmup)
    out = refine_poses(lab, dep, meta, r, p, pts, num_rows=num)
    active = int(out["icp_info"][:, 1:].abs().sum(1).gt(0).sum())

    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    net = vgg16_convs(num_classes=C, device=dev).init_random(seed=0, bias_std=0.05)
    rgb, _ = synth.make_images(B, H, W, seed=3)
    data, meta_n, ext = T(rgb), T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)), T(synth.extents_for(C))
    net.calibrate_background(data, meta_n, ext, dense_vertex=False)
    g0 = GraphedForward(net, data, meta_n, ext, dense_vertex=False)
    ms_off = time_ms(lambda: g0(data), args.steps, args.warmup)
    g1 = GraphedForward(net, data, meta_n, ext, dense_vertex=False, refine_depth=dep, refine_points=pts)
    ms_on = time_ms(lambda: g1(data, refine_depth=dep), args.steps, args.warmup)
    ms_off2 = time_ms(lambda: g0(data), args.steps, args.warmup)
    det = int(g1.layers["num_detections"].item())
    refined = int(g1.layers["detections_icp_info"][:, 1:].abs().sum(1).gt(0).sum())
    print(json.dumps(dict(bench="pose_refine", gpu=gpu_info(), batch=B, height=H, width=W, points=int(pts.shape[1]), rois=n,
                          rois_refined=active, refine_ms_per_batch=round(ms_refine, 4), refine_ms_per_roi=round(ms_refine / max(n, 1), 5),
                          graphed_ms_per_step_without_refine=round(min(ms_off, ms_off2), 3), graphed_ms_per_step_with_refine=round(ms_on, 3),
                          graphed_detections=det, graphed_rows_refined=refined, steps=args.steps, warmup=args.warmup)))


if __name__ == "__main__":
    main()
