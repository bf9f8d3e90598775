"""Time the training image blobs (posecnn_b200.augment) on the GPU, the host loader they replace, and the training step fed by them.

    python tools/bench_augment.py [--batch 64] [--iters 50] [--steps 10] [--cpu-frames 16] [--out FILE]

1. Device ms per batch at 640 x 480 for augment_color (lov_color_2d.yml draws: background, chromatic, noise) and depth_blob_train,
   CUDA events around each launch with L2 flushed before it; achieved GB/s against the compulsory traffic (colour: rgba 4 +
   background 3 + blob 12 bytes per pixel; depth: u16 2 read twice + blob 12).
2. The reference's host path on the same frames: composite + cv2 chromatic_transform + add_noise + mean subtraction, one thread and
   a process per core (only when cv2 is importable).
3. Trainer.step frames/s with the colour blob formed in the step against resident uint8 frames, alternating.
The card's name and power limit are printed with the numbers.
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

MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, iters, flush):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for s, e in ev:
        flush.zero_()
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    t = sorted(s.elapsed_time(e) for s, e in ev)
    return t[len(t) // 2], t[0]


# ---- the reference's host path, restated with the same cv2 / numpy calls (lib/utils/blob.py:74-129, minibatch.py:157-180)
def _host_frame(args):
    import cv2
    rgba, bg, seed = args
    rs = np.random.RandomState(seed)
    im = np.copy(rgba[:, :, :3])
    I = np.where(rgba[:, :, 3] == 0)
    im[I[0], I[1], :] = bg[I[0], I[1], :3]
    d_h = (rs.rand(1) - 0.5) * 0.02 * 180
    d_l = (rs.rand(1) - 0.5) * 0.2 * 256
    d_s = (rs.rand(1) - 0.5) * 0.2 * 256
    h, l, s = cv2.split(cv2.cvtColor(im, cv2.COLOR_BGR2HLS))
    new = cv2.merge(((h + d_h) % 180, np.clip(l + d_l, 0, 255), np.clip(s + d_s, 0, 255))).astype("uint8")
    im = cv2.cvtColor(new, cv2.COLOR_HLS2BGR)
    if rs.rand(1) < 0.9:
        sigma = (rs.rand(1) * 0.3 * 256) ** 0.5
        g = sigma * rs.randn(*im.shape[:2])
        im = np.clip(im + np.repeat(g[:, :, None], 3, axis=2), 0, 255)
    else:
        size = (3, 5, 7, 9, 11, 15)[int(rs.randint(6, size=1)[0])]
        k = np.zeros((size, size))
        if rs.rand(1) < 0.5:
            k[(size - 1) // 2, :] = 1
        else:
            k[:, (size - 1) // 2] = 1
        im = cv2.filter2D(im, -1, k / size)
    out = im.astype(np.float32, copy=True)
    out -= MEANS
    return out


def _init_worker():
    import cv2
    cv2.setNumThreads(1)


def host_rates(rgba, bg, n):
    try:
        import cv2  # noqa: F401
    except ImportError:
        return None
    import multiprocessing as mp
    work = [(rgba[i % len(rgba)], bg[i % len(bg)], i) for i in range(n)]
    _init_worker()
    _host_frame(work[0])
    t = time.perf_counter()
    for w in work:
        _host_frame(w)
    one = (time.perf_counter() - t) / n
    cores = os.cpu_count()
    with mp.get_context("fork").Pool(cores, initializer=_init_worker) as pool:
        pool.map(_host_frame, work[:cores])
        t = time.perf_counter()
        pool.map(_host_frame, work * max(1, cores // 4), chunksize=1)
        allc = (time.perf_counter() - t) / (n * max(1, cores // 4))
    return dict(ms_per_frame_1_thread=one * 1e3, frames_per_s_1_thread=1 / one, cores=cores, frames_per_s_all_cores=1 / allc)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--cpu-frames", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_augment needs a CUDA device")
    from posecnn_b200 import augment
    dev = torch.device("cuda:0")
    B, H, W = a.batch, 480, 640
    g = np.random.default_rng(0)
    rgba = g.integers(0, 256, (B, H, W, 4), dtype=np.uint8)
    rgba[..., 3] = np.where(g.random((B, H, W)) < 0.6, 0, 255)
    bgs = g.integers(0, 256, (8, H, W, 3), dtype=np.uint8)
    depth = g.integers(300, 4000, (B, H, W), dtype=np.uint16)
    x, pool = torch.from_numpy(rgba).to(dev), augment.background_pool(list(bgs)).to(dev)
    d = torch.from_numpy(depth.view(np.int16)).to(dev).view(torch.uint16)
    params, keys = augment.draw_params(np.random.RandomState(1), B, len(bgs), device=dev)
    dparams, dkeys = augment.draw_params(np.random.RandomState(2), B, 0, depth=True, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(5):
        augment.augment_color(x, pool, params, keys)
        augment.depth_blob_train(d, dparams, dkeys)
    c_med, c_min = timed(lambda: augment.augment_color(x, pool, params, keys), a.iters, flush)
    d_med, d_min = timed(lambda: augment.depth_blob_train(d, dparams, dkeys), a.iters, flush)
    px = B * H * W
    res = dict(card=card(), batch=B, height=H, width=W,
               color_ms=c_med, color_ms_min=c_min, color_GBps=px * 19 / (c_med * 1e-3) / 1e9,
               depth_ms=d_med, depth_ms_min=d_min, depth_GBps=px * 16 / (d_med * 1e-3) / 1e9)
    res["host_reference"] = host_rates(rgba[:8], bgs, a.cpu_frames)
    # training step: uint8 frames resident vs the colour blob formed inside the step (reported per frame)
    if a.steps > 0:
        from posecnn_b200.networks.vgg16_convs import vgg16_convs
        from posecnn_b200.train import Trainer
        from tools.bench_train_rgbd import C, make_inputs
        (rgb, *rest), _ = make_inputs(dev, B)                    # the seeded scene of bench.py --workload train
        net = vgg16_convs(num_classes=C, device=dev, is_train=True, fold_vertex_head=False).init_random(seed=0)
        tr = Trainer(net)
        data = rgb
        frames = torch.cat([rgb, torch.full_like(rgb[..., :1], 255)], 3).contiguous()   # the same frames with an opaque alpha
        u8 = lambda: tr.step(data, *rest)
        aug = lambda: tr.step(augment.augment_color(frames, pool, params, keys), *rest)
        for f in (u8, aug):
            f()
        times = {"u8": [], "aug": []}
        for _ in range(a.steps):
            for name, f in (("u8", u8), ("aug", aug)):
                torch.cuda.synchronize()
                t = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t)
        for name, v in times.items():
            res[f"step_{name}_ms"] = float(np.median(v) * 1e3)
            res[f"step_{name}_frames_per_s"] = B / float(np.median(v))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
