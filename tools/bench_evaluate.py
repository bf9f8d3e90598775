"""Cost of the device evaluator (DESIGN.md §14) at batch 32, 640x480, C = 22, five objects per image, three pose sets:
the confusion kernel (ms, GB/s against the 8 bytes per pixel it must read), the pose-error entry (ms, pairs/s) and the float64 /
scipy oracle on the host for the same batch (ms).  Prints one JSON line with the card and its power limit read in the same run.

    python tools/bench_evaluate.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from posecnn_b200 import synth  # noqa: E402
from posecnn_b200.evaluate import LOV_EVAL_SYMMETRIC, Evaluator  # noqa: E402
from tests import eval_ref  # noqa: E402

SETS = ("poses", "poses_refined", "poses_icp")


def batch(B, H, W, C, per_image, seed=0):
    """Coherent label maps and five detected objects per image (one detection each) with three noisy pose sets."""
    rng = np.random.default_rng(seed)
    gt = np.zeros((B, H, W), np.int32)
    rows, rois, poses = [], [], [[], [], []]
    for b in range(B):
        classes = rng.choice(np.arange(1, C), per_image, replace=False)
        for cls in classes:
            y, x = rng.integers(0, H - 120), rng.integers(0, W - 160)
            gt[b, y:y + 100, x:x + 120] = cls
            q = synth._rand_quat(rng)
            t = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.1, 0.1), rng.uniform(0.6, 1.2)])
            RT = eval_ref.estimate_rt(np.r_[q, t])
            rows.append(np.r_[b, cls, RT.reshape(-1)])
            rois.append([b, cls, x, y, x + 120, y + 100, 1.0])
            for s in range(3):
                qn, tn = synth.perturb_pose(q, t, rng, angle_deg=3.0 * (s + 1), lateral=0.005, depth=0.01)
                poses[s].append(np.r_[qn, tn])
    pred = np.where(rng.random((B, H, W)) < 0.03, rng.integers(0, C, (B, H, W)), gt).astype(np.int32)
    return gt, pred, np.array(rows, np.float32), np.array(rois, np.float32), np.array(poses, np.float32)


def gpu_ms(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--host-reps", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate needs a CUDA device")
    B, H, W, C, per = 32, 480, 640, 22, 5
    dev = torch.device("cuda:0")
    gt, pred, rows, rois, poses = batch(B, H, W, C, per)
    pts = synth.make_model_points(C, 2620)
    ext = synth.extents_for(C)
    meta = np.stack([synth.make_meta(synth.intrinsics(H, W))] * B).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ev = Evaluator(C, pts, ext, LOV_EVAL_SYMMETRIC, pose_sets=SETS, device=dev)
    g, p = T(gt), T(pred)
    ms_hist = gpu_ms(lambda: ev.add_labels(g, p), args.iters)
    pargs = (T(rows), T(rois), {s: T(poses[i]) for i, s in enumerate(SETS)}, torch.tensor([rois.shape[0]], dtype=torch.int32, device=dev),
             T(meta))
    ms_pose = gpu_ms(lambda: ev.add_poses(*pargs), max(args.iters // 4, 10))
    out = ev.add_poses(*pargs)
    npairs = int(out["num_pairs"].item())
    # correctness at the timed size: the device against the oracle
    ref = eval_ref.score(rows, rois, list(poses), rois.shape[0], meta, pts, LOV_EVAL_SYMMETRIC, eval_ref.default_threshold(ext),
                         np.zeros(C, np.float32), C)
    err = np.abs(out["errors"][:, :npairs].cpu().numpy() - ref[1]).max(axis=(0, 1))
    t0 = time.perf_counter()
    for _ in range(args.host_reps):
        eval_ref.fast_hist(gt.reshape(-1), pred.reshape(-1), C)
        eval_ref.score(rows, rois, list(poses), rois.shape[0], meta, pts, LOV_EVAL_SYMMETRIC, eval_ref.default_threshold(ext),
                       np.zeros(C, np.float32), C)
    host_ms = (time.perf_counter() - t0) * 1e3 / args.host_reps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    npx = B * H * W
    print(json.dumps(dict(
        card=smi, batch=B, height=H, width=W, num_classes=C, objects_per_image=per, pose_sets=len(SETS), points=pts.shape[1],
        confusion_ms=round(ms_hist, 4), confusion_GBps=round(8 * npx / (ms_hist * 1e-3) / 1e9, 1),
        pose_errors_ms=round(ms_pose, 4), pairs=npairs, pair_sets_per_s=round(npairs * len(SETS) / (ms_pose * 1e-3), 0),
        host_oracle_ms=round(host_ms, 1), max_abs_err_vs_oracle=[float(x) for x in err])))


if __name__ == "__main__":
    main()
