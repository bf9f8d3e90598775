"""Device time of the reference's OWN CUDA kernels (oracle/_ref, compiled unmodified for sm_90a) next to this repo's,
on the same inputs: Houghvotinggpu (one 640x480x22 frame and batch 4), RoiPool, Hardlabel.  Context for BASELINE.md:
the reference publishes no numbers; this is what its code does on the GPU it runs on."""
import json, os, sys, time
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref
from posecnn_b200 import synth
from posecnn_b200.build import build_native
build_native()
from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as hop
from posecnn_b200.hard_label_layer import hard_label_op as hlop
from posecnn_b200.roi_pooling_layer import roi_pooling_op as rop
assert ref.available(), "oracle/_ref/libposecnn_ref.so missing"
dev = torch.device("cuda:0")
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
rows = []


def wall(fn, n=3):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        torch.cuda.synchronize(); t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


for B in (1, 4):
    sc = synth.make_scene(batch=B, height=480, width=640, num_classes=22, seed=1234)
    d = [T(sc[k]) for k in ("label", "vertex", "extents", "meta")]
    t_ref = wall(lambda: ref.hough_full(*d, None, 0, -1.0, 0.02, 10), n=2)
    t_our = wall(lambda: hop.hough_voting_gpu_capacity(*d, None, 0, -1.0, 0.02, 10), n=10)
    rows.append(dict(op=f"Houghvotinggpu B={B} 640x480x22", reference_ms=t_ref, ours_ms=t_our, speedup=t_ref / t_our))
rng = np.random.default_rng(0)
feat = T(rng.standard_normal((32, 60, 80, 512)).astype(np.float32)); rois = T(synth.make_rois(128, 32, seed=5))
t_ref = wall(lambda: ref.roi_pool(feat, rois, 7, 7, 1 / 8.0)); t_our = wall(lambda: rop.roi_pool(feat, rois, 7, 7, 1 / 8.0), n=10)
rows.append(dict(op="RoiPool fwd conv4_3 N=128", reference_ms=t_ref, ours_ms=t_our, speedup=t_ref / t_our))
top, arg = rop.roi_pool(feat, rois, 7, 7, 1 / 8.0); g = torch.randn_like(top)
t_ref = wall(lambda: ref.roi_pool_grad(feat, rois, arg, g, 7, 7, 1 / 8.0)); t_our = wall(lambda: rop.roi_pool_grad(feat, rois, arg, g, 7, 7, 1 / 8.0), n=10)
rows.append(dict(op="RoiPoolGrad conv4_3 N=128 B=32", reference_ms=t_ref, ours_ms=t_our, speedup=t_ref / t_our))
prob = torch.rand((8, 480, 640, 22), device=dev); gt = torch.randint(-1, 22, (8, 480, 640), device=dev, dtype=torch.int32)
t_ref = wall(lambda: ref.hard_label(prob, gt, 1.0)); t_our = wall(lambda: hlop.hard_label(prob, gt, 1.0), n=10)
rows.append(dict(op="Hardlabel B=8", reference_ms=t_ref, ours_ms=t_our, speedup=t_ref / t_our))
for r in rows:
    print(f"{r['op']:36s} reference kernels {r['reference_ms']:10.3f} ms   this repo {r['ours_ms']:8.3f} ms   x{r['speedup']:.1f}")
print("(wall clock around synchronised calls incl. launch overhead and, for the reference Hough, its host round trips)")
