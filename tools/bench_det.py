"""Time the detection network (vgg16_det, lov_det.yml: C = 22, A = 20) at test time on the GPU.

    python tools/bench_det.py [--batches 1 32] [--iters 20] [--out FILE]

For each batch size at 480 x 640: the forward ms/step eager and graph-replayed (CUDA events over --iters steps after warm-up);
the proposal stage alone, per kernel (rpn_heads, rpn_select, rpn_nms_mask, rpn_nms_scan) from torch.profiler's CUDA kernel
times; and fc6's achieved TFLOP/s (2 * rows * 25088 * 4096 over the call's time, GEMM + epilogue).  The card's name and power limit are printed
with the numbers.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def events_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def kernel_ms(fn, iters, names):
    """Mean device ms per call of each kernel whose name contains one of `names` (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                out[n] += ev.device_time_total / 1000.0 / iters
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_det.py measures on the GPU"
    from posecnn_b200 import pose_head, synth
    from posecnn_b200.networks.vgg16_det import GraphedForward, vgg16_det
    dev = torch.device("cuda:0")
    net = vgg16_det(num_classes=22, device=dev).init_random(seed=0, bias_std=0.05)
    res = {"card": card(), "shape": "480x640", "C": 22, "A": net.num_anchors, "batches": {}}
    for B in args.batches:
        rgb, _ = synth.make_images(B, 480, 640, seed=B)
        data = torch.from_numpy(np.ascontiguousarray(rgb)).to(dev)
        fwd = lambda: net.forward(data, sync_rois=False)
        for _ in range(3):
            fwd()
        eager = events_ms(fwd, args.iters)
        g = GraphedForward(net, data)
        graphed = events_ms(lambda: g(data), args.iters)
        L = net.forward(data, sync_rois=False)
        from posecnn_b200.rpn_layer.proposal_layer import proposal_layer, rpn_heads
        rpn = L["conv_rpn"]
        T = net._tc
        anchors = net.anchors(30, 40)
        stage = lambda: proposal_layer(*rpn_heads(rpn, T["rpn/weights"], T["rpn/biases"], net.num_anchors), (480, 640, 1.0), "TEST",
                                       16, anchors, net.num_anchors)
        for _ in range(3):
            stage()
        per_kernel = kernel_ms(stage, args.iters, ["k_rpn_heads", "k_rpn_select", "k_rpn_nms_mask", "k_rpn_nms_scan"])
        stage_ms = events_ms(stage, args.iters)
        x = pose_head.crop_pool(L["conv5_3"], L["rois"], 16.0)
        fc6 = lambda: pose_head.fc(x, T["fc6/weights"], net.params["fc6/biases"], "relu")
        fc6()
        fc6_ms = events_ms(fc6, args.iters)
        rows = x.shape[0]
        res["batches"][B] = dict(forward_ms_eager=eager, forward_ms_graphed=graphed, proposal_stage_ms=stage_ms,
                                 proposal_kernels_ms=per_kernel, fc6_ms=fc6_ms, fc6_rows=rows,
                                 fc6_tflops=2.0 * rows * 25088 * 4096 / (fc6_ms * 1e-3) / 1e12,
                                 kept_per_image=L["num_rois"].tolist()[:4])
        print(B, json.dumps(res["batches"][B]), flush=True)
        del g
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
