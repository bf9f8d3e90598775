"""Time the object-coordinate pose estimator (csrc/coord_pose.cu, DESIGN.md §13): one call on a batch of analytic 640x480 scenes
(C = 22, three objects per image, 2 mm coordinate noise, 20 % outlier pixels), CUDA events over `--iters` calls after warm-up.
Also the per-kernel device time (torch.profiler, separate pass) and the GraphedForward step of a VERTEX_REG_3D network with and
without estimation.  Prints the card's name and power limit with the numbers, one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import synth
from posecnn_b200.coord_pose import estimate_poses_3d


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
    for _ in range(args.warmup):
        out = estimate_poses_3d(*inp, vertex=vertex)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        out = estimate_poses_3d(*inp, vertex=vertex)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.iters
    objects = int((out["info"][..., 1] > 0).sum())
    # per-kernel device time, in a separate profiled pass
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            estimate_poses_3d(*inp, vertex=vertex)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        for name in ("k_lists", "k_sample", "k_ransac"):
            if name in ev.key:
                kernels[name] = round(ev.device_time_total / 1000.0 / 5, 3)
    # GraphedForward step of a VERTEX_REG_3D network (random weights) with and without estimation
    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    net = vgg16_convs(num_classes=C, device=dev, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False).init_random(seed=0,
                                                                                                                   bias_std=0.05)
    rgb, depth_m = synth.make_images(B, 480, 640, seed=3)
    data = T(rgb)
    meta = T(np.stack([synth.make_meta(synth.intrinsics(480, 640))] * B))
    depth = T((depth_m * 10000.0).astype(np.float32))
    step = {}
    for tag, kw in (("without", {}), ("with", dict(estimate_depth=depth))):
        gf = GraphedForward(net, data, meta, inp[3], dense_vertex=False, **kw)
        for _ in range(args.warmup):
            gf(data, meta)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.iters):
            gf(data, meta)
        e1.record()
        torch.cuda.synchronize()
        step[tag] = round(e0.elapsed_time(e1) / args.iters, 3)
        del gf
    print(json.dumps(dict(workload="coord_pose3d", card=card, batch=B, num_classes=C, height=480, width=640, objects=objects,
                          ms_per_batch=round(ms, 3), ms_per_object=round(ms / max(objects, 1), 4), kernel_ms=kernels,
                          graphed_forward_ms=step)))


if __name__ == "__main__":
    main()
