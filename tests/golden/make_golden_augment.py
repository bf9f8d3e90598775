"""Generate tests/golden/augment.npz by EXECUTING THE REFERENCE'S OWN `chromatic_transform` and `add_noise`
(lib/utils/blob.py:74-129).  The module is Python 2, so each function's source text is cut out of the file unmodified, its tabs
expanded to 8 columns as Python 2 reads them (add_noise has one tab-indented line), and exec'd with `np` and `cv2`.

Each case seeds numpy's global RandomState and runs the loader's image path (minibatch.py:157-180): composite the background where
alpha == 0, chromatic_transform, add_noise, im.astype(float32) - PIXEL_MEANS.  The oracle (tests/augment_ref.py) recovers the
draws by replaying the same RandomState sequence.  Small images are stored whole; 480 x 640 blobs as a SHA-256 of their bytes.
Depth cases run add_noise on d / max(d) * 255 tiled x3 (minibatch.py:187-197).

    python tests/golden/make_golden_augment.py        # needs /root/reference and cv2; the .npz is committed
"""
import hashlib
import os
import re
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import augment_ref as ref  # noqa: E402

PIXEL_MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])         # lib/fcn/config.py:242


def reference_functions():
    src = open("/root/reference/lib/utils/blob.py").read().expandtabs(8)
    ns = dict(np=np, cv2=cv2)
    for name in ("chromatic_transform", "add_noise"):
        m = re.search(r"^def %s\(.*?(?=^def |\Z)" % name, src, re.S | re.M)
        exec(m.group(0), ns)
    return ns["chromatic_transform"], ns["add_noise"]


def inputs(H, W, seed):
    """A frame: random colours, alpha 0 on a band of rows and a scatter of pixels; a background; a raw depth image (u16)."""
    g = np.random.default_rng(seed)
    rgba = g.integers(0, 256, (H, W, 4), dtype=np.uint8)
    rgba[..., 3] = np.where(g.random((H, W)) < 0.3, 0, rgba[..., 3] | 1)
    rgba[: H // 4, :, 3] = 0
    bg = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    depth = g.integers(0, 4000, (H, W), dtype=np.uint16)
    return rgba, bg, depth


def noise_branch(seed, H, W, chromatic):
    rs = np.random.RandomState(seed)
    if chromatic:
        ref.replay_chromatic(rs)
    cols, _ = ref.replay_add_noise(rs, H, W)
    return (cols[0], cols[2], cols[3]) if cols[0] == ref.NOISE_BLUR else (cols[0],)


def seeds_covering(H, W, chromatic, want):
    """The first seeds whose add_noise draws hit each wanted branch in order: ('gauss',) or (size, axis); a branch may repeat."""
    seeds, s = [], 0
    for k in want:
        while True:
            b = noise_branch(s, H, W, chromatic)
            s += 1
            if k == (("gauss",) if b[0] == ref.NOISE_GAUSS else (int(b[1]), int(b[2]))):
                seeds.append(s - 1)
                break
    return seeds


def main():
    chromatic_transform, add_noise = reference_functions()
    cv2.setNumThreads(1)
    out = {}
    blur_all = [(z, a) for z in ref.BLUR_SIZES for a in (0, 1)]
    # colour, small frames: every blur size and orientation and three Gaussian draws, stored whole
    H, W = 20, 28
    seeds = seeds_covering(H, W, True, [("gauss",)] * 3 + blur_all)
    small = []
    for i, s in enumerate(seeds):
        rgba, bg, _ = inputs(H, W, 100 + i)
        np.random.seed(s)
        im = np.copy(rgba[:, :, :3])
        I = np.where(rgba[:, :, 3] == 0)
        im[I[0], I[1], :] = bg[I[0], I[1], :3]
        im = chromatic_transform(im)
        im = add_noise(im)
        blob = im.astype(np.float32, copy=True)
        blob -= PIXEL_MEANS
        small.append((s, rgba, bg, blob))
    out.update(small_seed=np.array([c[0] for c in small]), small_rgba=np.stack([c[1] for c in small]),
               small_bg=np.stack([c[2] for c in small]), small_blob=np.stack([c[3] for c in small]))
    # colour, 480 x 640: two Gaussian frames, a 15-tap blur (cv2's DFT path) along each axis and a 3-tap blur; digests
    H, W = 480, 640
    big_seeds = seeds_covering(H, W, True, [("gauss",), ("gauss",), (15, 0), (15, 1), (3, 1)])
    digests = []
    for i, s in enumerate(big_seeds):
        rgba, bg, _ = inputs(H, W, 200 + i)
        np.random.seed(s)
        im = np.copy(rgba[:, :, :3])
        I = np.where(rgba[:, :, 3] == 0)
        im[I[0], I[1], :] = bg[I[0], I[1], :3]
        im = add_noise(chromatic_transform(im))
        blob = im.astype(np.float32, copy=True)
        blob -= PIXEL_MEANS
        digests.append(hashlib.sha256(np.ascontiguousarray(blob).tobytes()).hexdigest())
    out.update(big_seed=np.array(big_seeds), big_input_seed=200 + np.arange(len(big_seeds)), big_sha256=np.array(digests))
    # depth, small frames: the float image through add_noise (Gaussian exact; cv2's float filter2D is compared within a tolerance)
    H, W = 20, 28
    dseeds = seeds_covering(H, W, False, [("gauss",), (3, 0), (15, 1), (9, 0)])
    dep = []
    for i, s in enumerate(dseeds):
        _, _, d = inputs(H, W, 300 + i)
        np.random.seed(s)
        im_depth = d.astype(np.float32, copy=True) / float(d.max()) * 255
        im_depth = np.tile(im_depth[:, :, np.newaxis], (1, 1, 3))
        im_depth = add_noise(im_depth)
        blob = im_depth.astype(np.float32, copy=True)
        blob -= PIXEL_MEANS
        dep.append((s, d, blob))
    out.update(depth_seed=np.array([c[0] for c in dep]), depth_raw=np.stack([c[1] for c in dep]), depth_blob=np.stack([c[2] for c in dep]))
    path = os.path.join(ROOT, "tests", "golden", "augment.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", len(small), "small,", len(big_seeds), "480x640,", len(dep), "depth cases")


if __name__ == "__main__":
    main()
