"""Roofline table of the memory-bound hot-path ops (SURVEY.md §8(d) algorithmic bytes / CUDA-event time)."""
import json, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import synth
from posecnn_b200.build import build_native
build_native()
from posecnn_b200.average_distance_loss import average_distance_loss_op as aop
from posecnn_b200.backprojecting_layer import backprojecting_op as bop
from posecnn_b200.hard_label_layer import hard_label_op as hop
from posecnn_b200.projecting_layer import projecting_op as pop
from posecnn_b200.roi_pooling_layer import roi_pooling_op as rop

dev = torch.device("cuda:0")
pk = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 6650.0
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
rows = []


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def report(name, ms, nbytes, note=""):
    gbs = nbytes / ms / 1e6
    rows.append(dict(op=name, ms=ms, algorithmic_bytes=nbytes, gbs=gbs, frac_of_measured_hbm=gbs / pk, note=note))
    print(f"{name:34s} {ms:8.3f} ms  {nbytes/1e6:9.1f} MB  {gbs:8.0f} GB/s  {gbs/pk*100:5.1f}% of {pk:.0f}  {note}")


B, H, W, C = 32, 480, 640, 22
# Hardlabel: gt + one prob + C outputs per pixel (compulsory), footprint 8C+4 B/px
prob = torch.rand((B, H, W, C), device=dev); gt = torch.randint(-1, C, (B, H, W), device=dev, dtype=torch.int32)
ms = timeit(lambda: hop.hard_label(prob, gt, 1.0))
report("hard_label fwd B32", ms, B * H * W * (4 + 4 + 4 * C), "compulsory bytes (gt + 1 prob + C out); footprint %.0f MB" % (B * H * W * (8 * C + 4) / 1e6))
del prob
# RoiPool fwd: 128 rois on conv5_3 / conv4_3 (bf16 trunk features and fp32)
rois = torch.from_numpy(synth.make_rois(128, B, seed=5)).to(dev)
for nm, h, w, sc in (("conv5_3", 30, 40, 1 / 16.0), ("conv4_3", 60, 80, 1 / 8.0)):
    f32 = torch.randn((B, h, w, 512), device=dev); bf = f32.to(torch.bfloat16)
    r = rois.cpu().numpy()
    area = 0
    for x1, y1, x2, y2 in r[:, 2:6]:
        a = (min(round(x2 * sc), w - 1) - max(round(x1 * sc), 0) + 1) * (min(round(y2 * sc), h - 1) - max(round(y1 * sc), 0) + 1)
        area += max(a, 0)
    out_b = 128 * 49 * 512 * 8
    ms = timeit(lambda: rop.roi_pool(f32, rois, 7, 7, sc, 0)); report(f"roi_pool fwd f32 {nm} N128", ms, area * 512 * 4 + out_b, "touched bin area + outputs")
    ms = timeit(lambda: rop.roi_pool(bf, rois, 7, 7, sc, 0)); report(f"roi_pool fwd bf16 {nm} N128", ms, area * 512 * 2 + out_b, "touched bin area + outputs")
    top, arg = rop.roi_pool(f32, rois, 7, 7, sc, 0); g = torch.randn_like(top)
    ms = timeit(lambda: rop.roi_pool_grad(f32, rois, arg, g, 7, 7, sc, 0)); report(f"roi_pool bwd {nm} N128", ms, B * h * w * 512 * 4 + out_b, "dense grad write + pooled reads")
    del f32, bf
# pose head (csrc/fc_tc.cu): fused RoiPool pair -> fc6 -> fc7 -> fc8 at 128 ROI rows; weight streaming, HBM bound
from posecnn_b200 import pose_head
f5 = torch.randn((B, 30, 40, 512), device=dev).to(torch.bfloat16); f4 = torch.randn((B, 60, 80, 512), device=dev).to(torch.bfloat16)
r = rois.cpu().numpy(); area = 0
for (h, w, sc) in ((30, 40, 1 / 16.0), (60, 80, 1 / 8.0)):
    for x1, y1, x2, y2 in r[:, 2:6]:
        area += max((min(round(x2 * sc), w - 1) - max(round(x1 * sc), 0) + 1) * (min(round(y2 * sc), h - 1) - max(round(y1 * sc), 0) + 1), 0)
ms = timeit(lambda: pose_head.roi_pool_pair(f5, f4, rois)); report("roi_pool_pair bf16 (conv5_3 + conv4_3) N128", ms, area * 512 * 2 + 128 * 49 * 512 * 2, "touched bin areas + bf16 fc6 operand")
xa = pose_head.roi_pool_pair(f5, f4, rois)
for nm, K, N in (("fc6", 25088, 4096), ("fc7", 4096, 4096), ("fc8", 4096, 88)):
    wt = pose_head.fc_weights_to_tc(torch.randn((K, N), device=dev) * 0.01); bs = torch.zeros(N, device=dev)
    a = xa if K == 25088 else torch.randn((128, K), device=dev).to(torch.float16)
    ms = timeit(lambda: pose_head.fc(a, wt, bs, "relu" if N > 88 else "tanh", torch.float16 if N > 88 else torch.float32))
    report(f"{nm} 128 x {K} x {N} fp16 (split-K wgmma + finish)", ms, wt.numel() * 2 + 128 * K * 2 + 128 * N * 4, "weights + A + out; 2*M*K*N = %.1f GFLOP" % (2 * 128 * K * N / 1e9))
    del wt
del f5, f4, xa
# Project / Backproject, G = 128, Cf = 64, batch 4 (8.6 GB of voxel grids at batch 4)
Bp, G, Cf = 4, 128, 64
case = synth.make_projection_case(Bp, H, W, Cf, 3, 8, seed=5)  # small grid for meta only
meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(H, W), G)] * Bp)).to(dev)
depth = torch.from_numpy(case["depth"]).to(dev)
vox = torch.randn((Bp, G, G, G, Cf), device=dev)
ms = timeit(lambda: pop.project(vox, depth, meta, 3, 0.02)); report(f"project fwd B{Bp} G{G} Cf{Cf}", ms, Bp * H * W * (4 + 8 * Cf), "B*H*W*(4 + 8 Cf)")
data = torch.randn((Bp, H, W, Cf), device=dev); lab = torch.rand((Bp, H, W, C), device=dev); l3 = torch.rand((Bp, G, G, G, C), device=dev)
ms = timeit(lambda: bop.backproject(data, lab, depth, meta, l3, G, 3, 0.02), n=3)
report(f"backproject fwd B{Bp} G{G} Cf{Cf}", ms, Bp * G**3 * (2 * Cf + C) * 4 + Bp * H * W * (Cf + C + 1) * 4, "B*G^3*(2Cf+C)*4 written + B*H*W*(Cf+C+1)*4 read")
del vox, l3, data, lab
# Averagedistance: N = 64*9 rois, P = 2620
pts = torch.from_numpy(synth.make_model_points(C, 2620)).to(dev); sym = torch.from_numpy(synth.LOV_SYMMETRY).to(dev)
pred, targ, wt = [torch.from_numpy(a).to(dev) for a in synth.make_pose_batch(576, C, seed=9)]
ms = timeit(lambda: aop.average_distance_loss(pred, targ, wt, pts, sym, 0.01))
nsym = int(sum(1 for n in range(576) if wt[n].any() and sym[int(torch.argmax(wt[n])) // 4] > 0))
report("average_distance fwd N576 P2620", ms, 576 * 4 * C * 12 + C * 2620 * 12, f"{nsym} symmetric rois (O(P^2) closest-point search, compute bound)")
nact = int(sum(1 for n in range(576) if wt[n].any()))
flop = (nact - nsym) * 2620 * 60.0 + nsym * 2620.0 * 2620.0 * 20.0      # SURVEY 8(d): non-sym N*P*~60, sym N*P^2*~20
fp32_peak = 132 * 128 * 2 * 1.98e9 / 1e12                                # H100 SXM CUDA-core fp32 FMA peak at the max SM clock, TFLOP/s
rows[-1].update(flop=flop, tflops=flop / ms / 1e9, frac_of_fp32_peak=flop / ms / 1e9 / fp32_peak)
print(f"  average_distance FLOP view: {flop/1e9:.2f} GFLOP ({nsym} symmetric of {nact} active rois) -> {flop/ms/1e9:.2f} TFLOP/s = {flop/ms/1e9/fp32_peak*100:.1f}% of the {fp32_peak:.1f} TFLOP/s fp32 CUDA-core peak")
json.dump(rows, open(os.path.join(os.path.dirname(__file__), "..", "gpurun_out", "bench_ops.json"), "w"), indent=1)
