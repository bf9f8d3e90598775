"""The resize restatement (tests/rescale_ref.py) against OpenCV's generic build, and the argument checks of the rescale entries
(csrc/rescale.cu) without a GPU."""
import ctypes

import numpy as np
import pytest

from tests import rescale_ref as ref

SCALES = (1.5, 1.25, 2.0)
SHAPES = ((480, 640), (37, 53))


@pytest.fixture(scope="module")
def cv2_generic():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    yield cv2
    cv2.setUseOptimized(was)


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("hw", SHAPES)
@pytest.mark.parametrize("channels", [1, 3])
def test_linear_f32_equals_cv2(cv2_generic, s, hw, channels):
    g = np.random.default_rng(hash((s, hw, channels)) % 2 ** 32)
    shape = hw + ((channels,) if channels == 3 else ())
    x = ((g.random(shape) - 0.45) * 300).astype(np.float32)
    want = cv2_generic.resize(x, None, None, fx=s, fy=s, interpolation=cv2_generic.INTER_LINEAR)
    got = ref.resize_linear_f32(x, s)
    assert got.shape == want.shape == ref.scaled_size(*hw, s) + shape[2:]
    assert (u32(got) != u32(want)).sum() == 0


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("hw", SHAPES)
def test_linear_u16_equals_cv2(cv2_generic, s, hw):
    g = np.random.default_rng(7)
    d = g.integers(0, 65536, hw).astype(np.uint16)
    d[: hw[0] // 4] = g.integers(400, 1200, (hw[0] // 4, hw[1]))        # sensor-like range next to full-range noise
    d[hw[0] // 2, : hw[1] // 2] = 0                                      # holes
    want = cv2_generic.resize(d, None, None, fx=s, fy=s, interpolation=cv2_generic.INTER_LINEAR)
    assert np.array_equal(ref.resize_linear_u16(d, s), want)


def test_color_blob_equals_cv2(cv2_generic):
    """lib/fcn/test.py:49-65 as the reference writes it: im.astype(float32) - PIXEL_MEANS (float64), cv2.resize LINEAR."""
    g = np.random.default_rng(2)
    im = g.integers(0, 256, (480, 640, 3), dtype=np.uint8)
    orig = im.astype(np.float32, copy=True)
    orig -= ref.PIXEL_MEANS
    want = cv2_generic.resize(orig, None, None, fx=1.5, fy=1.5, interpolation=cv2_generic.INTER_LINEAR)
    assert (u32(ref.color_blob(im, 1.5)) != u32(want)).sum() == 0


@pytest.mark.parametrize("s", [1.5, 1.0 / 1.5])
@pytest.mark.parametrize("dtype", [np.int32, np.uint8])
@pytest.mark.parametrize("hw", [(480, 640), (720, 960), (37, 53)])
def test_nearest_equals_cv2(cv2_generic, s, dtype, hw):
    g = np.random.default_rng(5)
    x = g.integers(0, 22, hw).astype(dtype)
    want = cv2_generic.resize(x, None, None, fx=s, fy=s, interpolation=cv2_generic.INTER_NEAREST)
    assert np.array_equal(ref.resize_nearest(x, s), want)


def test_round_trip_sizes():
    assert ref.scaled_size(480, 640, 1.5) == (720, 960)
    assert ref.scaled_size(720, 960, 1.0 / 1.5) == (480, 640)
    assert ref.scaled_size(37, 53, 1.5) == (56, 80)            # 55.5 and 79.5: half to even
    from posecnn_b200 import rescale
    for H, W, s in ((480, 640, 1.5), (37, 53, 1.5), (37, 53, 1.25), (45, 61, 2.0), (720, 960, 1 / 1.5)):
        assert rescale.scaled_size(H, W, s) == ref.scaled_size(H, W, s)
    for bad in (0.0, -1.5, float("inf"), float("nan")):
        with pytest.raises(ValueError):
            rescale.scaled_size(480, 640, bad)


def test_optimized_build_deviation_is_recorded():
    """The reference's output depends on its OpenCV build: the default (SIMD) build rounds differently from the generic one that
    rescale.cu reproduces.  Printed, not bounded."""
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(True)
    try:
        g = np.random.default_rng(0)
        im = g.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        orig = im.astype(np.float32) - ref.PIXEL_MEANS.astype(np.float32)
        opt = cv2.resize(orig.astype(np.float32), None, None, fx=1.5, fy=1.5, interpolation=cv2.INTER_LINEAR)
        d = g.integers(300, 3000, (480, 640)).astype(np.uint16)
        dopt = cv2.resize(d, None, None, fx=1.5, fy=1.5, interpolation=cv2.INTER_LINEAR)
    finally:
        cv2.setUseOptimized(was)
    e = np.abs(opt - ref.resize_linear_f32(orig.astype(np.float32), 1.5)).max()
    du = np.abs(dopt.astype(np.int64) - ref.resize_linear_u16(d, 1.5).astype(np.int64))
    print(f"cv2 {cv2.__version__} optimized build vs generic at s = 1.5: colour blob max |diff| {e:.3e}; depth "
          f"{(du != 0).mean() * 100:.2f} % of pixels differ, max {du.max()}")


def test_rescale_entries_reject_bad_arguments_without_gpu(native_lib):
    mean = (ctypes.c_double * 3)(102.9801, 115.9465, 122.7717)
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    lin, col, dep, nn = (native_lib.pcnn_resize_linear_f32, native_lib.pcnn_resize_color_u8, native_lib.pcnn_resize_depth,
                         native_lib.pcnn_resize_nearest_i32)
    err = lambda: native_lib.pcnn_last_error()
    # NULL pointers and channel counts
    assert lin(None, 1, 480, 640, 3, 1.5, 720, 960, buf, None) == -1 and b"NULL" in err()
    assert col(buf, 1, 480, 640, 1.5, 720, 960, None, buf, None) == -1 and b"NULL" in err()
    assert dep(buf, 1, 1, 480, 640, 1.5, 720, 960, None, None) == -1 and b"NULL" in err()
    assert nn(buf, 1, 480, 640, 1.5, 720, 960, None, None) == -1 and b"NULL" in err()
    assert lin(buf, 1, 480, 640, 2, 1.5, 720, 960, buf, None) == -1 and b"C must be 1 or 3" in err()
    # bad shapes and factors
    for B, H, W in ((0, 480, 640), (1, 0, 640), (1, 480, -1), (65536, 480, 640)):
        assert nn(buf, B, H, W, 1.5, 720, 960, buf, None) == -1, (B, H, W)
    for fx in (0.0, -1.5, float("inf"), float("nan")):
        assert dep(buf, 1, 1, 480, 640, fx, 720, 960, buf, None) == -1 and b"fx" in err()
    assert nn(buf, 1, 480, 640, 1e-4, 0, 0, buf, None) == -1 and b"empty" in err()
    # the destination size must be cv2's round(H fx) x round(W fx), half to even
    for Ho, Wo in ((721, 960), (720, 959), (480, 640)):
        assert col(buf, 1, 480, 640, 1.5, Ho, Wo, mean, buf, None) == -1 and b"round" in err()
    assert nn(buf, 2, 37, 53, 1.5, 55, 79, buf, None) == -1 and b"56 x 80" in err()
    assert nn(buf, 2, 720, 960, 1.0 / 1.5, 479, 640, buf, None) == -1 and b"480 x 640" in err()
    # rows whose flat in-row index would overflow int are refused, before any launch
    W = (1 << 31) // 3 + 1
    assert lin(buf, 1, 1, W, 3, 1.0, 1, W, buf, None) == -1 and b"overflow" in err()
    assert col(buf, 1, 1, W, 1.0, 1, W, mean, buf, None) == -1 and b"overflow" in err()
    W = (1 << 30)
    assert lin(buf, 1, 1, W, 1, 2.0, 2, 2 * W, buf, None) == -1 and b"too large" in err()
