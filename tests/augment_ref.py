"""numpy restatement of the training image blobs (posecnn_b200.augment / csrc/augment.cu), the tests' oracle.

It restates, step by step, what the reference's loader does per image (lib/gt_synthesize_layer/minibatch.py:147-200,
lib/utils/blob.py:74-129), with OpenCV's uint8 HLS conversions emulated in float32:
  - BGR -> HLS (RGB2HLS_f's vector form): s = diff / (l < 0.5 ? vmax + vmin : 2 - (vmax + vmin)); the hue is ONE fused multiply-add
    x * (60 / diff) + c with c = 360 (red maximum, x < 0), 0, 120 or 240; outputs rounded half to even;
  - HLS -> BGR: the scalar sector table of HLS2RGB_f (hscale 6 / 180);
both equal cv2.cvtColor on every input (tests/test_augment_cpu.py checks all 2^24 colours and all 181 * 256 * 256 HLS triples).
The Gaussian field is Philox4x32-10 + Box-Muller, the same generator as the kernel.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
PIXEL_MEANS = np.array([102.9801, 115.9465, 122.7717])           # lib/fcn/config.py:242
NOISE_NONE, NOISE_GAUSS, NOISE_BLUR = 0, 1, 2
BLUR_SIZES = (3, 5, 7, 9, 11, 15)


# ---------------------------------------------------------------- random numbers
def philox4x32_10(key: int, ctr: np.ndarray):
    """Philox4x32-10 on counters (ctr as u64 -> words 0, 1; words 2, 3 = 0) with a 64-bit key; returns the four u32 words."""
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    mask = np.uint64(0xFFFFFFFF)
    ctr = np.asarray(ctr, np.uint64)
    c0, c1 = ctr & mask, ctr >> np.uint64(32)
    c2 = np.zeros_like(c0)
    c3 = np.zeros_like(c0)
    k0, k1 = int(key) & 0xFFFFFFFF, (int(key) >> 32) & 0xFFFFFFFF
    for i in range(10):
        if i:
            k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
    return c0, c1, c2, c3


def philox_normal(key: int, H: int, W: int) -> np.ndarray:
    """The kernel's Gaussian field of one image [H, W] f64: Box-Muller on u1 in (0, 1], u2 in [0, 1) (53 bits each)."""
    c0, c1, c2, c3 = philox4x32_10(key, np.arange(H * W, dtype=np.uint64))
    s = np.uint64(32)
    u1 = (((c0 << s) | c1) >> np.uint64(11)).astype(np.float64)
    u1 = (u1 + 1.0) * 2.0 ** -53
    u2 = (((c2 << s) | c3) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(6.283185307179586 * u2)).reshape(H, W)


# ---------------------------------------------------------------- OpenCV's uint8 HLS conversions
def _fma32(a, b, c):
    """fmaf(a, b, c) for float32 arrays: the exact product in f64, the sum rounded to odd in f64, then rounded to f32."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = np.broadcast_to(np.asarray(c, np.float64), p.shape)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    fix = (err != 0) & ((s.view(np.int64) & 1) == 0)
    return np.where(fix, np.nextafter(s, s + err), s).astype(F32)


def bgr2hls(img: np.ndarray) -> np.ndarray:
    """cv2.cvtColor(img, cv2.COLOR_BGR2HLS) for uint8 [..., 3]."""
    f = img.astype(F32) * F32(1 / 255.)
    b, g, r = f[..., 0], f[..., 1], f[..., 2]
    vmax = np.maximum(np.maximum(r, g), b)
    vmin = np.minimum(np.minimum(r, g), b)
    diff, msum = vmax - vmin, vmax + vmin
    l = msum * F32(0.5)
    with np.errstate(all="ignore"):
        s = diff / np.where(l < F32(0.5), msum, F32(2) - msum)
        inv = F32(60) / diff
        x = np.where(vmax == r, g - b, np.where(vmax == g, b - r, r - g))
        c = np.where(vmax == r, np.where(x < 0, F32(360), F32(0)), np.where(vmax == g, F32(120), F32(240)))
        h = _fma32(x, inv, c)
    ok = diff > np.finfo(F32).eps
    h, s = np.where(ok, h, F32(0)), np.where(ok, s, F32(0))
    out = [np.rint(h * F32(0.5)), np.rint(l * F32(255)), np.rint(s * F32(255))]
    return np.stack(out, -1).clip(0, 255).astype(np.uint8)


_SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def hls2bgr(hls: np.ndarray) -> np.ndarray:
    """cv2.cvtColor(hls, cv2.COLOR_HLS2BGR) for uint8 [..., 3] (hue 0..180)."""
    h = hls[..., 0].astype(F32)
    l = hls[..., 1].astype(F32) * F32(1 / 255.)
    s = hls[..., 2].astype(F32) * F32(1 / 255.)
    p2 = np.where(l <= F32(0.5), l * (F32(1) + s), (l + s) - l * s).astype(F32)
    p1 = (F32(2) * l - p2).astype(F32)
    hh = (h * (F32(6) / F32(180))).astype(F32)
    hh = np.where(hh >= F32(6), hh - F32(6), hh).astype(F32)
    sec = np.floor(hh).astype(np.int64)
    fr = (hh - sec.astype(F32)).astype(F32)
    d = p2 - p1
    tab = np.stack([p2, p1, p1 + d * (F32(1) - fr), p1 + d * fr], -1)
    bgr = [np.take_along_axis(tab, _SECTORS[sec][..., k:k + 1], -1)[..., 0] for k in range(3)]
    bgr = [np.where(s == 0, l, v) for v in bgr]
    return np.stack([np.rint(v * F32(255)) for v in bgr], -1).clip(0, 255).astype(np.uint8)


def chromatic(im: np.ndarray, d_h: float, d_l: float, d_s: float) -> np.ndarray:
    """chromatic_transform (blob.py:74-99) with given shifts."""
    hls = bgr2hls(im).astype(np.float64)
    new = np.stack([np.mod(hls[..., 0] + d_h, 180), np.clip(hls[..., 1] + d_l, 0, 255), np.clip(hls[..., 2] + d_s, 0, 255)], -1)
    return hls2bgr(new.astype(np.uint8))


# ---------------------------------------------------------------- noise
def _reflect101(i: np.ndarray, n: int) -> np.ndarray:
    if n == 1:
        return np.zeros_like(i)
    i = i.copy()
    while ((i < 0) | (i >= n)).any():
        i = np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i))
    return i


def _taps(x: np.ndarray, size: int, axis: int):
    """The blur's taps x[reflect101(p + t)], t = -r..r, along image axis `axis` (0 = along the row: x; 1 = along the column: y)."""
    r = (size - 1) // 2
    ax = 1 if axis == 0 else 0
    n = x.shape[ax]
    idx = np.arange(n)
    return [np.take(x, _reflect101(idx + t, n), axis=ax) for t in range(-r, r + 1)]


def blur_u8(im: np.ndarray, size: int, axis: int) -> np.ndarray:
    """cv2.filter2D(im, -1, motion kernel) on uint8: round(sum / size) (never a tie: size is odd)."""
    s = sum(t.astype(np.int64) for t in _taps(im, size, axis))
    return ((2 * s + size) // (2 * size)).astype(np.uint8)


def blur_f32(im: np.ndarray, size: int, axis: int) -> np.ndarray:
    """The kernel's blur on float data: the f64 sum of the taps in ascending order, / size, rounded once to f32."""
    s = np.zeros(im.shape, np.float64)
    for t in _taps(im, size, axis):
        s = s + t.astype(np.float64)
    return (s / size).astype(F32)


def _noise(x: np.ndarray, row, field) -> np.ndarray:
    """add_noise with the table row's parameters and the given [H, W] field -> f32 values."""
    mode = int(row[5])
    if mode == NOISE_GAUSS:
        g = (row[6] * field)[..., None]                              # one field for every channel (np.repeat, blob.py:113-114)
        with np.errstate(invalid="ignore"):
            return np.clip(x.astype(np.float64) + g, 0, 255).astype(F32)
    if mode == NOISE_BLUR:
        return blur_u8(x, int(row[7]), int(row[8])).astype(F32) if x.dtype == np.uint8 else blur_f32(x, int(row[7]), int(row[8]))
    return x.astype(F32)


def _field(key, field, b, H, W, mode):
    if mode != NOISE_GAUSS:
        return None
    return field[b] if field is not None else philox_normal(int(key), H, W)


# ---------------------------------------------------------------- blobs
def color_blob(rgba: np.ndarray, backgrounds, table: np.ndarray, keys, field=None) -> np.ndarray:
    """rgba [B,H,W,4|3] u8, backgrounds [N,H,W,3] u8 or None, table [B,9] -> blob [B,H,W,3] f32."""
    B, H, W, ch = rgba.shape
    n_bg = 0 if backgrounds is None else len(backgrounds)
    out = np.empty((B, H, W, 3), F32)
    for b in range(B):
        row = table[b]
        im = rgba[b, :, :, :3].copy()
        if ch == 4:
            bg = int(row[0]) if 0 <= row[0] < n_bg else -1
            I = rgba[b, :, :, 3] == 0
            im[I] = backgrounds[bg][I] if bg >= 0 else 0
        if row[1]:
            im = chromatic(im, row[2], row[3], row[4])
        x = _noise(im, row, _field(keys[b], field, b, H, W, int(row[5])))
        out[b] = (x.astype(np.float64) - PIXEL_MEANS).astype(F32)   # im_orig -= cfg.PIXEL_MEANS on a float32 array
    return out


def depth_blob(depth: np.ndarray, table: np.ndarray, keys, field=None):
    """depth [B,H,W] u16 / f32 -> (blob [B,H,W,3] f32, max [B] f32): d / max(d) * 255 tiled x3, add_noise, - PIXEL_MEANS."""
    B, H, W = depth.shape
    out = np.empty((B, H, W, 3), F32)
    mx = np.empty(B, F32)
    for b in range(B):
        mx[b] = F32(depth[b].max())
        with np.errstate(invalid="ignore", divide="ignore"):
            v = (depth[b].astype(F32) / mx[b]) * F32(255)
        x = _noise(v[..., None], table[b], _field(keys[b], field, b, H, W, int(table[b][5])))
        out[b] = (np.broadcast_to(x, (H, W, 3)).astype(np.float64) - PIXEL_MEANS).astype(F32)
    return out, mx


def replay_add_noise(rs: np.random.RandomState, H: int, W: int):
    """Replays add_noise's RandomState calls (blob.py:105-127): returns (table columns 5..8, field or None)."""
    r = rs.rand(1)
    if r < 0.9:
        var = rs.rand(1) * 0.3 * 256
        sigma = var ** 0.5
        return [NOISE_GAUSS, float(sigma[0]), 0.0, 0.0], rs.randn(H, W)
    size = BLUR_SIZES[int(rs.randint(len(BLUR_SIZES), size=1)[0])]
    axis = 0.0 if rs.rand(1) < 0.5 else 1.0
    return [NOISE_BLUR, 0.0, float(size), axis], None


def replay_chromatic(rs: np.random.RandomState):
    """Replays chromatic_transform's three draws (blob.py:78-83): (d_h, d_l, d_s)."""
    d_h = (rs.rand(1) - 0.5) * 0.02 * 180
    d_l = (rs.rand(1) - 0.5) * 0.2 * 256
    d_s = (rs.rand(1) - 0.5) * 0.2 * 256
    return float(d_h[0]), float(d_l[0]), float(d_s[0])
