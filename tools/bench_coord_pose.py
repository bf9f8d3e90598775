"""Time the object-coordinate pose estimators (csrc/coord_pose.cu, DESIGN.md §13), with depth (estimate_poses_3d) and colour only
(estimate_poses_2d): one call on a batch of analytic 640x480 scenes (C = 22, three objects per image, 2 mm coordinate noise, 20 %
outlier pixels), CUDA events over `--iters` calls after warm-up.  Also the per-kernel device time (torch.profiler, separate pass)
and the GraphedForward step of a VERTEX_REG_3D network without estimation, with estimate_depth and with estimate_rgb.  Prints the
card's name and power limit with the numbers, one JSON line per estimator."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import synth
from posecnn_b200.coord_pose import estimate_poses_2d, estimate_poses_3d


def timed(fn, warmup, iters):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, out


def kernel_ms(fn, names):
    """Per-kernel device time of one call (torch.profiler over 5 calls)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        for name in names:
            if name + "<" in ev.key or name + "(" in ev.key:
                kernels[name] = round(kernels.get(name, 0.0) + ev.device_time_total / 1000.0 / 5, 3)
    return kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_coord_pose needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    B, C = args.batch, 22
    sc = synth.make_coordinate_scene(batch=B, num_classes=C, seed=101, coord_noise_m=0.002, outlier_fraction=0.2)
    dev = torch.device("cuda")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    keys = torch.arange(1, B + 1, dtype=torch.int64, device=dev) * 7919
    inp = (T(sc["label"]), T(sc["depth"]), T(sc["meta"]), T(sc["extents"]), keys)
    vertex = T(sc["vertex"])
    f3 = lambda: estimate_poses_3d(*inp, vertex=vertex)
    f2 = lambda: estimate_poses_2d(inp[0], inp[2], inp[3], keys, vertex=vertex)
    res = {}
    for tag, fn, names in (("coord_pose3d", f3, ("k_lists", "k_sample", "k_ransac")),
                           ("coord_pose2d", f2, ("k_lists", "k_sample2d", "k_ransac"))):
        ms, out = timed(fn, args.warmup, args.iters)
        objects = int((out["info"][..., 1] > 0).sum())
        res[tag] = dict(objects=objects, ms_per_batch=round(ms, 3), ms_per_object=round(ms / max(objects, 1), 4),
                        kernel_ms=kernel_ms(fn, names))
    # GraphedForward step of a VERTEX_REG_3D network (random weights) with and without estimation
    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    net = vgg16_convs(num_classes=C, device=dev, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False).init_random(seed=0,
                                                                                                                   bias_std=0.05)
    rgb, depth_m = synth.make_images(B, 480, 640, seed=3)
    data = T(rgb)
    meta = T(np.stack([synth.make_meta(synth.intrinsics(480, 640))] * B))
    depth = T((depth_m * 10000.0).astype(np.float32))
    step = {}
    for tag, kw in (("without", {}), ("with", dict(estimate_depth=depth)), ("with_rgb", dict(estimate_rgb=True))):
        gf = GraphedForward(net, data, meta, inp[3], dense_vertex=False, **kw)
        step[tag] = round(timed(lambda: gf(data, meta), args.warmup, args.iters)[0], 3)
        del gf
    for tag, r in res.items():
        step_tag = dict(coord_pose3d=("without", "with"), coord_pose2d=("without", "with_rgb"))[tag]
        print(json.dumps(dict(workload=tag, card=card, batch=B, num_classes=C, height=480, width=640, **r,
                              graphed_forward_ms={"without": step[step_tag[0]], "with": step[step_tag[1]]})))


if __name__ == "__main__":
    main()
