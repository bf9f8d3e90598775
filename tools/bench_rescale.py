"""Time the image-scale resizes (posecnn_b200.rescale) and the object-coordinate network at the resolution SCALES_BASE 1.5 gives.

    python tools/bench_rescale.py [--batch 32] [--iters 50] [--steps 10] [--out FILE]

1. Each resize at batch 32, 480 x 640 -> 720 x 960: CUDA events around each launch with L2 flushed before it (median of --iters);
   bytes = compulsory traffic (source read once, destination written once) over time, and its share of the H100 SXM data sheet's
   3.35 TB/s.
2. GraphedForward of a random-weight vertex_reg_3d network (C = 2, the LINEMOD configuration) at batch 32, at 720 x 960 against
   480 x 640, without and with estimate_depth (the pose estimate from object coordinates and depth): median replay time.
3. The C = 2 object-coordinate training step (Trainer.step with vertmap) at batch 2 (IMS_PER_BATCH of linemod_*_3d.yml) and 32, at
   both sizes: median of --steps steps after two warm-up steps, host clock around a device synchronise.
A workload that does not fit in device memory is reported as "not measured (out of memory)".  The card's name, power limit and
maximum SM clock are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BPS = 3.35e12          # H100 SXM HBM3, data sheet
S = 1.5


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, iters, flush=None):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for s, e in ev:
        if flush is not None:
            flush.zero_()
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    t = sorted(s.elapsed_time(e) for s, e in ev)
    return t[len(t) // 2]


def resizes(dev, B, iters):
    from posecnn_b200 import rescale
    H, W = 480, 640
    Ho, Wo = rescale.scaled_size(H, W, S)
    g = torch.Generator(device=dev).manual_seed(0)
    frames = torch.randint(0, 256, (B, H, W, 3), generator=g, device=dev, dtype=torch.uint8)
    x3 = torch.randn(B, H, W, 3, generator=g, device=dev)
    d32 = torch.randint(300, 4000, (B, H, W), generator=g, device=dev).float()
    d16 = d32.to(torch.int32).to(torch.int16).view(torch.uint16)
    lab = torch.randint(0, 2, (B, H, W), generator=g, device=dev, dtype=torch.int32)
    cases = {   # name: (call, bytes per source pixel read, bytes per destination pixel written)
        "color_blob_u8": (lambda: rescale.color_blob(frames, S), 3, 12),
        "resize_linear_f32_c3": (lambda: rescale.resize_linear(x3, S), 12, 12),
        "resize_depth_u16": (lambda: rescale.resize_depth(d16, S), 2, 2),
        "resize_depth_f32": (lambda: rescale.resize_depth(d32, S), 4, 4),
        "resize_nearest_i32": (lambda: rescale.resize_nearest(lab, S), 4, 4),
    }
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = {}
    for name, (fn, rb, wb) in cases.items():
        for _ in range(3):
            fn()
        ms = timed(fn, iters, flush)
        nbytes = B * (H * W * rb + Ho * Wo * wb)
        out[name] = dict(ms=ms, bytes=nbytes, GBps=nbytes / (ms * 1e-3) / 1e9, share_of_3_35_TBps=nbytes / (ms * 1e-3) / PEAK_BPS)
    return out


def net_inputs(dev, B, H, W, C):
    from posecnn_b200 import synth
    rgb, depth_m = synth.make_images(min(B, 2), H, W, seed=3)
    rep = lambda a: np.ascontiguousarray(np.concatenate([a] * ((B + a.shape[0] - 1) // a.shape[0]))[:B])
    T = lambda a: torch.from_numpy(rep(a)).to(dev)
    meta = T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * min(B, 2)))
    return T(rgb), T(np.rint(depth_m * 10000.0).astype(np.float32)), meta, torch.from_numpy(synth.extents_for(C)).to(dev)


def forward(dev, B, iters):
    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    C = 2
    net = vgg16_convs(num_classes=C, device=dev, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False,
                      scales=(S,)).init_random(seed=0, bias_std=0.05)
    res = {}
    for H, W in ((480, 640), (720, 960)):
        data, depth, meta, ext = net_inputs(dev, B, H, W, C)
        keys = torch.arange(B, dtype=torch.int64, device=dev)
        for est in (False, True):
            name = f"{H}x{W}" + ("_estimate_depth" if est else "")
            try:
                kw = dict(estimate_depth=depth, estimate_keys=keys) if est else {}
                gf = GraphedForward(net, data, meta, ext, dense_vertex=False, **kw)
                call = (lambda: gf(data, meta, estimate_depth=depth)) if est else (lambda: gf(data, meta))
                for _ in range(3):
                    call()
                ms = timed(call, iters)
                res[name] = dict(ms=ms, frames_per_s=B / (ms * 1e-3))
                del gf
            except torch.cuda.OutOfMemoryError:
                res[name] = "not measured (out of memory)"
            torch.cuda.empty_cache()
    return res


def train(dev, batches, steps):
    from posecnn_b200 import synth
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.train import Trainer
    C = 2
    res = {}
    for H, W in ((480, 640), (720, 960)):
        sc = synth.make_coordinate_scene(batch=2, height=H, width=W, num_classes=C, objects_per_image=1, seed=11)
        for B in batches:
            name = f"{H}x{W}_batch{B}"
            rep = lambda a: torch.from_numpy(np.ascontiguousarray(np.concatenate([a] * (B // 2))[:B])).to(dev)
            rgb, _ = synth.make_images(2, H, W, seed=3)
            cen = np.zeros((2, C, 3), np.float32)
            cen[:, 1, 2] = 1.0
            meta = np.stack([synth.make_meta(synth.intrinsics(H, W)).reshape(48)] * 2)
            args = (rep(rgb), rep(sc["label"]), rep(cen), rep(meta), torch.from_numpy(sc["extents"]).to(dev),
                    torch.zeros((0, 13), device=dev), torch.from_numpy(synth.make_model_points(C, 50)).to(dev), torch.zeros(C, device=dev))
            vm = rep(sc["coords"])
            try:
                net = vgg16_convs(num_classes=C, device=dev, is_train=True, fold_vertex_head=False, vertex_reg_2d=False, vertex_reg_3d=True,
                                  pose_reg=False).init_random(seed=0, bias_std=0.02)
                tr = Trainer(net, lr=1e-6, vertex_w=10.0, vertex_w_inside=10.0)
                for _ in range(2):
                    tr.step(*args, vertmap=vm)
                t = []
                for _ in range(steps):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    tr.step(*args, vertmap=vm)
                    torch.cuda.synchronize()
                    t.append(time.perf_counter() - t0)
                ms = float(np.median(t) * 1e3)
                res[name] = dict(ms=ms, frames_per_s=B / (ms * 1e-3))
                del tr, net
            except torch.cuda.OutOfMemoryError:
                res[name] = "not measured (out of memory)"
            torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rescale needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(card=card(), scale=S)
    res["resize_batch%d_480x640_to_720x960" % a.batch] = resizes(dev, a.batch, a.iters)
    res["graphed_forward_vertex_reg_3d_C2_batch%d" % a.batch] = forward(dev, a.batch, max(5, a.iters // 5))
    res["train_step_vertex_reg_3d_C2"] = train(dev, (2, a.batch), a.steps)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
