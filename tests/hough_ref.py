"""Helpers of the exactness tests of Houghvotinggpu (tests/test_hough_exact_gpu.py, tests/test_hough_slack_cpu.py).

* `band_rows` restates the band height rule of csrc/hough_vote.cu, so that each test asserts which k_vote band height
  (16, 8, 4, 2 or 1 rows: lane rotation `(lane + k) & (R - 1)` and band / row bookkeeping) it covers.
* `check_planes` is the exactness criterion of the interval scan (DESIGN.md §3.3): the device plane equals the oracle's
  plane wherever no irregular (sample, row) pair reaches the cell, and differs by at most the slack elsewhere.  A pair is
  irregular where the reference's fp32 predicate is not one interval along the window row (the own row: not one whole
  side); the oracle counts them (`oracle.hough_voting_gpu(..., slack=True)`).
* scene builders: the scenes the `hough` benchmark workload votes on, and small planted scenes for the predicate's edges.
"""
import math

import numpy as np

from posecnn_b200 import synth

NUM_SMS = 132              # kNumSMs (csrc/common.cuh)
BAND_MIN_ROWS = 8          # PCNN_HOUGH_BAND_MIN default
BENCH_SEED = 2234          # bench.py hough_scenes(0): 1234 + 1000 * config 1
BENCH_FRAMES = 8


def band_rows(B, H, W, C):
    """k_vote's band height (band_rows in csrc/hough_vote.cu): 16 rows while R x (W + 3) ints fit 48 KB of shared memory,
    halved for wider images; halved down to 8 rows while B x C x ceil(H / R) is below 16 items per resident CTA."""
    R = 16
    while R > 1 and R * (W + 3) * 4 > 48 * 1024:
        R >>= 1
    while R > BAND_MIN_ROWS and B * C * math.ceil(H / R) < 16 * 4 * NUM_SMS:
        R >>= 1
    return R


def check_planes(got, dbg, what=""):
    """Criterion of DESIGN.md §3.3 on [B,C,H,W] planes: equal where the slack is 0, |difference| <= slack elsewhere.
    Returns a summary dict (cells that differ, pairs, irregular pairs)."""
    votes, slack = dbg["votes"], dbg["slack"]
    got = np.asarray(got)
    assert got.shape == votes.shape, (got.shape, votes.shape)
    diff = np.abs(got.astype(np.int64) - votes.astype(np.int64))
    exact = slack == 0
    bad_exact = exact & (diff > 0)
    if bad_exact.any():
        b, c, y, x = np.argwhere(bad_exact)[0]
        raise AssertionError(f"{what}: {int(bad_exact.sum())} cells without irregular pairs differ from the oracle; first at "
                             f"image {b} class {c} (x={x}, y={y}): {got[b, c, y, x]} vs {votes[b, c, y, x]}")
    over = diff > slack
    assert not over.any(), f"{what}: {int(over.sum())} cells differ by more than their slack (max diff {diff.max()})"
    pairs = dbg["pairs"].sum(axis=(0, 1))
    return dict(cells_differ=int((diff > 0).sum()), pairs=int(pairs[0]), irregular=int(pairs[1]),
                slack_cells=int((~exact).sum()), max_vote=int(votes.max()))


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def bench_scenes():
    """The 8 distinct 480 x 640 x 22-class scenes the `hough` benchmark workload tiles into its batches."""
    return synth.make_scene(batch=BENCH_FRAMES, height=480, width=640, num_classes=22, seed=BENCH_SEED)


def tile(sc, B):
    """Batch B of the scenes repeated in order (bench.py hough_inputs); gt rows are repeated with their batch index."""
    n = sc["label"].shape[0]
    reps = -(-B // n)
    t = lambda a: np.concatenate([a] * reps, 0)[:B]
    gt = sc["gt"]
    gts = [np.concatenate([gt[:, :1] + k * n, gt[:, 1:]], 1) for k in range(reps)]
    gt = np.concatenate(gts, 0)
    gt = np.ascontiguousarray(gt[gt[:, 0] < B], np.float32)
    return dict(sc, label=t(sc["label"]), vertex=t(sc["vertex"]), meta=t(sc["meta"]), gt=gt)


def blank_scene(B, H, W, C, f=None, seed=0):
    """Background-only scene: label 0, unit-variance noise in the vertex channels, a pinhole camera with focal length
    f (default: the YCB camera scaled to W) centred on the image."""
    rng = np.random.default_rng(seed)
    f = synth.FX * W / 640.0 if f is None else f
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], np.float64)
    meta = np.stack([synth.make_meta(K)] * B).reshape(B, 1, 1, 48)
    return dict(label=np.zeros((B, H, W), np.int32), vertex=rng.standard_normal((B, H, W, 3 * C), dtype=np.float32),
                extents=synth.extents_for(C), meta=meta, gt=np.zeros((0, 13), np.float32), rng=rng)


def plant(sc, b, cls, cx, cy, rx, ry, z, noise=0.05):
    """An elliptic object of class cls centred at (cx, cy) with radii (rx, ry): label, unit directions to the centre plus
    Gaussian noise, log depth z.  Returns the (ys, xs) of its pixels in raster order."""
    H, W = sc["label"].shape[1:]
    ys, xs = np.mgrid[0:H, 0:W]
    mask = ((xs - cx) / rx) ** 2 + ((ys - cy) / ry) ** 2 <= 1.0
    sc["label"][b][mask] = cls
    ys, xs = np.nonzero(mask)
    dx, dy = cx - xs, cy - ys
    n = np.sqrt(dx * dx + dy * dy) + 1e-10
    rng = sc["rng"]
    sc["vertex"][b, ys, xs, 3 * cls] = (dx / n + rng.normal(0, noise, xs.size)).astype(np.float32)
    sc["vertex"][b, ys, xs, 3 * cls + 1] = (dy / n + rng.normal(0, noise, xs.size)).astype(np.float32)
    sc["vertex"][b, ys, xs, 3 * cls + 2] = np.float32(np.log(z))
    return ys, xs


def norm_f32(u, v):
    """n1 = RN(sqrt(fma(u, u, RN(v * v)))) for directions of magnitude ~1 (the float64 sum is exact there)."""
    u, v = np.float32(u), np.float32(v)
    return np.sqrt(np.float32(np.float64(u) * np.float64(u) + np.float64(v * v)), dtype=np.float32)


def ratio_f32(u, v):
    """u / n1 as the reference rounds it."""
    return np.float32(np.float32(u) / norm_f32(u, v))


def near_threshold_dirs(k_ulps=4, inlier=0.9, seed=0, count=16):
    """Directions (u, v) whose rounded u / n1 lies k ulps (k = -k_ulps .. k_ulps) from float32(inlier), half of them
    mirrored to -u: on the pixel's own row the reference's cosine is RN(RN(u dx) / RN(n1 |dx|)), which these pixels put
    on either side of the threshold depending on dx."""
    rng = np.random.default_rng(seed)
    t = np.float32(inlier)
    out = []
    for i in range(count):
        v = np.float32(rng.uniform(0.3, 3.0)) * np.float32(1 if i % 2 else -1)
        u0 = np.float32(abs(float(v)) * inlier / math.sqrt(1 - inlier * inlier))
        for k in range(-k_ulps, k_ulps + 1):
            target = t
            for _ in range(abs(k)):
                target = np.nextafter(target, np.float32(2 if k > 0 else 0))
            u = u0
            for _ in range(400):
                r = ratio_f32(u, v)
                if r == target:
                    break
                u = np.nextafter(u, np.float32(1e3 if r < target else 0))
            if ratio_f32(u, v) == target:
                out.append((u, v) if i % 4 < 2 else (-u, v))
    return np.array(out, np.float32)
