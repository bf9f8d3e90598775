"""numpy restatement of OpenCV's generic (non-SIMD) cv2.resize, the arithmetic csrc/rescale.cu reproduces bit for bit.

LINEAR:  per destination index d, f = float32((d + 0.5) * (1 / s) - 0.5) computed in float64, sx = floor(f), a = f - sx in float32.
Columns: sx < 0 -> (0, a = 0), sx >= W - 1 -> (W - 1, a = 0), second tap min(sx + 1, W - 1).  Rows: only the row indices sy, sy + 1
are clamped to [0, H - 1]; the row weight b is never zeroed.  h = RN(RN(S0 (1 - a)) + RN(S1 a)), out = RN(RN(h0 (1 - b)) + RN(h1 b)),
every operation a float32 one.  uint16 output rounds half to even (rint) and saturates to [0, 65535].
NEAREST: sx = min(floor(d * (1 / s)), W - 1) in float64, s the caller's float64 factor.
Sizes: round(H s) x round(W s) with round half to even (cv2's saturate_cast<int>(double)).
"""
import numpy as np

PIXEL_MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])


def scaled_size(H, W, s):
    return int(np.rint(H * float(s))), int(np.rint(W * float(s)))


def _linear_coords(n_out, n_in, s, clamp_weight):
    d = np.arange(n_out, dtype=np.float64)
    f = ((d + 0.5) * (1.0 / float(s)) - 0.5).astype(np.float32)
    i0 = np.floor(f).astype(np.int64)
    a = (f - i0.astype(np.float32)).astype(np.float32)
    if clamp_weight:
        lo, hi = i0 < 0, i0 >= n_in - 1
        a[lo | hi] = 0
        i0 = np.where(lo, 0, np.where(hi, n_in - 1, i0))
        i1 = np.minimum(i0 + 1, n_in - 1)
    else:
        i1 = np.clip(i0 + 1, 0, n_in - 1)
        i0 = np.clip(i0, 0, n_in - 1)
    return i0, i1, a, (np.float32(1) - a).astype(np.float32)


def resize_linear_f32(x, s):
    """x [H,W] or [H,W,C] float32 (or any dtype, converted to float32 first) -> float32, cv2.INTER_LINEAR."""
    x = np.asarray(x, np.float32)
    H, W = x.shape[:2]
    Ho, Wo = scaled_size(H, W, s)
    x0, x1, a, a0 = _linear_coords(Wo, W, s, True)
    y0, y1, b, b0 = _linear_coords(Ho, H, s, False)
    ex = (slice(None),) + (None,) * (x.ndim - 2)
    ey = (slice(None), None) + (None,) * (x.ndim - 2)
    with np.errstate(invalid="ignore", over="ignore"):
        h = (x[:, x0] * a0[ex]).astype(np.float32) + (x[:, x1] * a[ex]).astype(np.float32)
        return (h[y0] * b0[ey]).astype(np.float32) + (h[y1] * b[ey]).astype(np.float32)


def round_u16(v):
    """saturate_cast<ushort>(float): rint, saturate; NaN -> 0."""
    v = np.asarray(v, np.float32)
    with np.errstate(invalid="ignore"):
        r = np.clip(np.rint(np.nan_to_num(v, nan=0.0)), 0, 65535)
    return r.astype(np.uint16)


def resize_linear_u16(x, s):
    """x [H,W] uint16 -> uint16, cv2.INTER_LINEAR (float arithmetic, then rint and saturate)."""
    return round_u16(resize_linear_f32(np.asarray(x).astype(np.float32), s))


def color_blob(frame_u8, s, mean=PIXEL_MEANS):
    """lib/fcn/test.py:49-65: f32(u8) - PIXEL_MEANS as numpy computes it (float64 means, rounded to float32), then LINEAR."""
    x = (np.asarray(frame_u8).astype(np.float32) - np.asarray(mean, np.float64).reshape(1, 1, 3)).astype(np.float32)
    return resize_linear_f32(x, s)


def resize_nearest(x, s):
    """x [H,W(,C)] of any dtype -> same dtype, cv2.INTER_NEAREST at the float64 factor s."""
    x = np.asarray(x)
    H, W = x.shape[:2]
    Ho, Wo = scaled_size(H, W, s)
    inv = 1.0 / float(s)
    sx = np.minimum(np.floor(np.arange(Wo, dtype=np.float64) * inv).astype(np.int64), W - 1)
    sy = np.minimum(np.floor(np.arange(Ho, dtype=np.float64) * inv).astype(np.int64), H - 1)
    return x[sy][:, sx]
