"""Time the detection network (vgg16_det, lov_det.yml: C = 22, A = 20) at test time on the GPU.

    python tools/bench_det.py [--batches 1 32] [--iters 20] [--out FILE]

For each batch size at 480 x 640: the forward ms/step eager and graph-replayed (CUDA events over --iters steps after warm-up);
the proposal stage alone, per kernel (rpn_heads, rpn_select, rpn_nms_mask, rpn_nms_scan) from torch.profiler's CUDA kernel
times; and fc6's achieved TFLOP/s (2 * rows * 25088 * 4096 over the call's time, GEMM + epilogue).  The card's name and power limit are printed
with the numbers.  Prints one JSON object.

The detection records (det_records.detection_records) at C = 22 (lov_det.yml) and C = 2 (linemod_*_det.yml, A = 30), both
with a 2,620-point table: the records stage alone on the network's own outputs, the graph-replayed forward with and without
it, the mean and largest number of objective evaluations per filled slot, and the host path the reference runs (selection,
then scipy's Nelder-Mead on a numpy objective per record, tests/det_post_ref.py) per image on this machine's CPU.
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


def host_records_ms(L, meta, points, images):
    """The reference's host path per image: de-normalise, decode, select, then scipy's Nelder-Mead on a numpy objective for
    each record (CPU wall time)."""
    import time

    from scipy.optimize import minimize

    from tests import det_post_ref as ref
    cls_prob, bbox_pred, rois, poses_tanh, num = (L[k].cpu().numpy() for k in ("cls_prob", "bbox_pred", "rois", "poses_tanh", "num_rois"))
    N = rois.shape[0] // num.shape[0]
    t0 = time.perf_counter()
    for b in range(images):
        rows = slice(b * N, b * N + int(num[b]))
        boxes = ref.class_boxes(rois[rows], ref.denormalise(bbox_pred[rows]), 480, 640)
        K = meta[b, :9].astype(np.float64).reshape(3, 3)
        for j, r in ref.select(cls_prob[rows], int(num[b])):
            R, rx, ry, w, h = ref.fit_inputs(boxes[r, 4 * j:4 * j + 4], poses_tanh[rows][r, 4 * j:4 * j + 4], points[j], K)
            minimize(lambda x: ref.objective(float(x[0]), R, rx, ry, points[j], K, w, h), 0.5, method="nelder-mead")
    return (time.perf_counter() - t0) * 1e3 / images


def bench_records(dev, C, A, B, iters):
    from posecnn_b200 import synth
    from posecnn_b200.det_records import detection_records
    from posecnn_b200.networks.vgg16_det import GraphedForward, vgg16_det
    net = vgg16_det(num_classes=C, anchor_scales=(4, 8, 16, 32) if A == 20 else (3, 4, 5, 6, 7, 8), device=dev)
    net.init_random(seed=C, bias_std=0.05).set_points(synth.make_model_points(C, 2620))
    rgb, _ = synth.make_images(B, 480, 640, seed=B)
    data = torch.from_numpy(np.ascontiguousarray(rgb)).to(dev)
    meta_np = np.stack([synth.make_meta(synth.intrinsics(480, 640))] * B).astype(np.float32)
    meta = torch.from_numpy(meta_np).to(dev)
    L = {k: v.clone() for k, v in net.forward(data, sync_rois=False, meta_data=meta).items()}
    stage = lambda: detection_records(L["cls_prob"], L["bbox_pred"], L["poses_tanh"], L["rois"], L["num_rois"], (480, 640), meta,
                                      net.points)
    for _ in range(3):
        stage()
    stage_ms = events_ms(stage, iters)
    g0 = GraphedForward(net, data)
    without = events_ms(lambda: g0(data), iters)
    del g0
    g1 = GraphedForward(net, data, meta_data=meta)
    with_records = events_ms(lambda: g1(data, meta), iters)
    del g1
    nfev = L["det_trace"][:, 1].cpu().numpy()
    filled = nfev > 0
    return dict(records_ms=stage_ms, forward_ms_graphed=without, forward_ms_graphed_with_records=with_records,
                records=int(filled.sum()), slots=int(nfev.size), nfev_mean=float(nfev[filled].mean()) if filled.any() else 0.0,
                nfev_max=int(nfev.max()), host_ms_per_image=host_records_ms(L, meta_np, net.points.cpu().numpy(), min(B, 4)))


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
    res["records"] = {}
    for C, A in ((22, 20), (2, 30)):
        for B in args.batches:
            res["records"][f"C{C}_B{B}"] = bench_records(dev, C, A, B, args.iters)
            print(f"records C = {C}, B = {B}", json.dumps(res["records"][f"C{C}_B{B}"]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
