"""Training-step time of the RGB-D network against the colour network, in one process on one GPU.

Both steps run on the seeded synthetic 640x480 scene of `bench.py --workload train` (22 classes, labels / centres / poses
from synth.make_scene(seed=4234), images from synth.make_images(seed=21)); the RGB-D step also reads that call's depth image
in millimetres, as `bench.py --workload rgbd` feeds it.  The two steps alternate, three runs each: every run is --warmup
untimed steps and --steps steps timed with CUDA events.  The RGB-D step adds a second trunk forward and backward, so the
trunk rate counts 2 trunks x 3 x 187.918 GFLOP per frame (forward, input-gradient and weight-gradient GEMMs) against 1 for
colour.  The card name and power limit are read in the same run with a read-only nvidia-smi query.  Batch 64 falls back to
32 only when 64 does not fit, and the JSON says so.

    python tools/bench_train_rgbd.py [--batch 64] [--steps 20] [--warmup 3] [--runs 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import synth                                     # noqa: E402
from posecnn_b200.networks.vgg16_convs import vgg16_convs         # noqa: E402
from posecnn_b200.train import Trainer                             # noqa: E402

H, W, C = 480, 640, 22
VGG_FLOP_PER_FRAME = 187.918e9


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return dict(name=name, power_limit=power)
    except Exception as e:                                       # the figure is still printed, without its card
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({type(e).__name__})")


def make_inputs(dev, B):
    """The scene of bench.py run_train, whole batch on one GPU, plus the depth image in millimetres."""
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
    rgb, depth = synth.make_images(B, H, W, seed=21)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    args = (T(rgb), T(label), T(centers), T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)), T(synth.extents_for(C)), T(gt),
            T(synth.make_model_points(C, 2620)), T(synth.LOV_SYMMETRY))
    return args, T((depth * 1000.0).astype(np.float32))


def make_trainer(dev, fmt):
    net = vgg16_convs(input_format=fmt, num_classes=C, device=dev, is_train=True, fold_vertex_head=False).init_random(seed=0)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02; net.params["fc8/weights"] *= 0.01
    net.prepare()
    return Trainer(net, lr=1e-4, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0, margin=0.01)


def timed_run(tr, args, kw, steps, warmup):
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        out = tr.step(*args, **kw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = tr.step(*args, **kw)
    e1.record()
    torch.cuda.synchronize()
    losses = [float(out[k].item()) for k in ("loss_cls", "loss_vertex", "loss_pose")]
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated(), losses


def measure(dev, B, a):
    args, depth = make_inputs(dev, B)
    trainers = {"COLOR": make_trainer(dev, "COLOR"), "RGBD": make_trainer(dev, "RGBD")}
    kws = {"COLOR": {}, "RGBD": dict(depth=depth)}
    res = {k: dict(ms=[], mem=0, losses=[]) for k in trainers}
    for _ in range(a.runs):
        for fmt, tr in trainers.items():
            ms, mem, losses = timed_run(tr, args, kws[fmt], a.steps, a.warmup)
            res[fmt]["ms"].append(ms)
            res[fmt]["mem"] = max(res[fmt]["mem"], mem)
            res[fmt]["losses"] = losses
            assert all(np.isfinite(losses)), (fmt, losses)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info()
    B, note = a.batch, None
    try:
        res = measure(dev, B, a)
    except torch.cuda.OutOfMemoryError:
        if B <= 32:
            raise
        note = f"batch {B} did not fit in {torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB; measured at batch 32"
        torch.cuda.empty_cache()
        B = 32
        res = measure(dev, B, a)
    out = dict(metric="training step, RGB-D vs colour network", batch=B, steps=a.steps, warmup=a.warmup, runs=a.runs, image=f"{W}x{H}",
               gpu=info["name"], power_limit=info["power_limit"])
    for fmt, trunks in (("COLOR", 1), ("RGBD", 2)):
        ms = statistics.median(res[fmt]["ms"])
        out[fmt.lower()] = dict(ms_per_step=ms, ms_per_step_runs=res[fmt]["ms"], frames_per_s=B / (ms * 1e-3),
                                max_memory_allocated_gib=res[fmt]["mem"] / 2**30,
                                trunk_tflops=trunks * 3 * VGG_FLOP_PER_FRAME * B / (ms * 1e-3) / 1e12,
                                losses=dict(zip(("cls", "vertex", "pose"), res[fmt]["losses"])))
    out["ratio_rgbd_over_color"] = out["rgbd"]["ms_per_step"] / out["color"]["ms_per_step"]
    if note:
        out["note"] = note
    print(json.dumps(out))


if __name__ == "__main__":
    main()
