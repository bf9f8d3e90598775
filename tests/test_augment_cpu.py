"""CPU checks of the training image blobs: the numpy oracle (tests/augment_ref.py) against vectors made by the reference's own
chromatic_transform / add_noise (tests/golden/augment.npz), its HLS conversions against cv2 on every input, the parameter draw,
and the argument checks of the two C ABI entries (they fail before any CUDA call)."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

from tests import augment_ref as ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment.npz")


def replay_table(seed, H, W, chromatic=True):
    """The parameter row and field the reference drew after np.random.seed(seed) (background given by the case itself)."""
    rs = np.random.RandomState(seed)
    row = np.zeros(9)
    if chromatic:
        row[1] = 1
        row[2:5] = ref.replay_chromatic(rs)
    cols, field = ref.replay_add_noise(rs, H, W)
    row[5:9] = cols
    return row, field


def test_oracle_equals_reference_small_frames():
    g = np.load(GOLD)
    seeds, rgba, bg, want = g["small_seed"], g["small_rgba"], g["small_bg"], g["small_blob"]
    H, W = rgba.shape[1:3]
    modes = set()
    for i, s in enumerate(seeds):
        row, field = replay_table(int(s), H, W)
        row[0] = 0
        modes.add((int(row[5]), int(row[7]), int(row[8])))
        got = ref.color_blob(rgba[i:i + 1], bg[i:i + 1], row[None], [0], None if field is None else field[None])
        np.testing.assert_array_equal(got[0].view(np.uint32), want[i].view(np.uint32), err_msg=f"seed {s}")
    assert {m for m in modes if m[0] == ref.NOISE_BLUR} == {(2, z, a) for z in ref.BLUR_SIZES for a in (0, 1)}
    assert (ref.NOISE_GAUSS, 0, 0) in modes


def test_oracle_equals_reference_full_frames():
    from tests.golden.make_golden_augment import inputs
    g = np.load(GOLD)
    for s, si, digest in zip(g["big_seed"], g["big_input_seed"], g["big_sha256"]):
        rgba, bg, _ = inputs(480, 640, int(si))
        row, field = replay_table(int(s), 480, 640)
        row[0] = 0
        got = ref.color_blob(rgba[None], bg[None], row[None], [0], None if field is None else field[None])
        assert hashlib.sha256(got[0].tobytes()).hexdigest() == str(digest), f"seed {s}, noise {row[5:]}"


def test_depth_oracle_against_reference():
    """Gaussian: exact.  Blur: the kernel's f64 box mean against cv2's float32 filter2D (DFT at 15 taps): within 2e-4 absolute
    (values 0..255; measured 3.1e-5)."""
    g = np.load(GOLD)
    H, W = g["depth_raw"].shape[1:]
    for s, d, want in zip(g["depth_seed"], g["depth_raw"], g["depth_blob"]):
        row, field = replay_table(int(s), H, W, chromatic=False)
        row[0] = -1
        got, mx = ref.depth_blob(d[None], row[None], [0], None if field is None else field[None])
        assert mx[0] == d.max()
        if row[5] == ref.NOISE_GAUSS:
            np.testing.assert_array_equal(got[0].view(np.uint32), want.view(np.uint32))
        else:
            np.testing.assert_allclose(got[0], want, rtol=0, atol=2e-4)


def test_depth_oracle_all_zero_image_is_nan():
    row = np.zeros(9)
    got, mx = ref.depth_blob(np.zeros((1, 4, 5), np.uint16), row[None], [0])
    assert mx[0] == 0 and np.isnan(got).all()


def test_hls_conversions_equal_cv2_on_every_input():
    cv2 = pytest.importorskip("cv2")
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], 1).astype(np.uint8).reshape(4096, 4096, 3)
    mism = (ref.bgr2hls(img) != cv2.cvtColor(img, cv2.COLOR_BGR2HLS)).reshape(-1, 3).sum(0)
    assert mism.tolist() == [0, 0, 0]
    # hue 180 is reachable: (0 + d_h) % 180 rounds to 180.0 for a tiny negative d_h
    H, L, S = np.meshgrid(np.arange(181), np.arange(256), np.arange(256), indexing="ij")
    hls = np.stack([H, L, S], -1).astype(np.uint8).reshape(181 * 256, 256, 3)
    mism = (ref.hls2bgr(hls) != cv2.cvtColor(hls, cv2.COLOR_HLS2BGR)).reshape(-1, 3).sum(0)
    assert mism.tolist() == [0, 0, 0]


def test_blur_u8_equals_cv2_filter2d():
    cv2 = pytest.importorskip("cv2")
    im = np.random.default_rng(0).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    for size in ref.BLUR_SIZES:
        for axis in (0, 1):
            k = np.zeros((size, size))
            if axis == 0:
                k[(size - 1) // 2, :] = 1
            else:
                k[:, (size - 1) // 2] = 1
            np.testing.assert_array_equal(ref.blur_u8(im, size, axis), cv2.filter2D(im, -1, k / size), err_msg=f"{size} {axis}")


def test_philox_known_answer():
    # Random123 known-answer vector philox4x32_10: ctr = 0, key = 0
    c = ref.philox4x32_10(0, np.zeros(1, np.uint64))
    assert [int(w[0]) for w in c] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


def test_draw_params_ranges():
    from posecnn_b200 import augment
    rs = np.random.RandomState(7)
    table, keys = augment.draw_params(rs, 2000, 5, device="cpu")
    t = table.numpy()
    assert t.shape == (2000, augment.NUM_PARAMS) and keys.dtype.is_signed and keys.shape == (2000,)
    assert set(np.unique(t[:, 0])) <= set(range(5)) and (t[:, 1] == 1).all()
    assert (np.abs(t[:, 2]) <= 0.01 * 180).all() and (np.abs(t[:, 3:5]) <= 0.1 * 256).all()
    gauss, blur = t[:, 5] == augment.NOISE_GAUSS, t[:, 5] == augment.NOISE_BLUR
    assert (gauss | blur).all() and 0.86 < gauss.mean() < 0.94
    assert (t[gauss, 6] >= 0).all() and (t[gauss, 6] <= (0.3 * 256) ** 0.5).all()
    assert set(np.unique(t[blur, 7])) == set(augment.BLUR_SIZES) and set(np.unique(t[blur, 8])) == {0, 1}
    # the draw order is the reference's: replaying the same RandomState gives the same scalars
    rs = np.random.RandomState(7)
    for b in range(3):
        assert rs.randint(5, size=1)[0] == t[b, 0]
        assert np.allclose(ref.replay_chromatic(rs), t[b, 2:5], rtol=0, atol=0)
        r = rs.rand(1)
        if r < 0.9:
            assert ((rs.rand(1) * 0.3 * 256) ** 0.5)[0] == t[b, 6]
        else:
            assert ref.BLUR_SIZES[int(rs.randint(6, size=1)[0])] == t[b, 7]
            assert (0 if rs.rand(1) < 0.5 else 1) == t[b, 8]
    plain, _ = augment.draw_params(np.random.RandomState(1), 4, 0, chromatic=False, add_noise=False, device="cpu")
    assert (plain.numpy()[:, 0] == -1).all() and (plain.numpy()[:, 1:] == 0).all()
    with pytest.raises(ValueError):
        augment.validate_params(np.array([[7, 1, 0, 0, 0, 0, 0, 0, 0]], float), 5)
    with pytest.raises(ValueError):
        augment.validate_params(np.array([[-1, 1, 0, 0, 0, 2, 0, 4, 0]], float), 5)


def test_augment_entries_reject_bad_arguments_without_gpu(native_lib):
    native_lib.pcnn_last_error.restype = ctypes.c_char_p
    mean = (ctypes.c_double * 3)(102.9801, 115.9465, 122.7717)
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    f = native_lib.pcnn_augment_color_fwd
    assert f(None, 4, None, 0, buf, buf, None, 1, 8, 8, mean, buf, None) == -1
    assert b"NULL" in native_lib.pcnn_last_error()
    assert f(buf, 4, None, 0, buf, buf, None, 1, 8, 8, None, buf, None) == -1
    assert f(buf, 5, None, 0, buf, buf, None, 1, 8, 8, mean, buf, None) == -1
    assert b"channels" in native_lib.pcnn_last_error()
    assert f(buf, 4, None, 2, buf, buf, None, 1, 8, 8, mean, buf, None) == -1
    assert b"background" in native_lib.pcnn_last_error()
    for B, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -1), (65536, 8, 8)):
        assert f(buf, 3, None, 0, buf, buf, None, B, H, W, mean, buf, None) == -1, (B, H, W)
    g = native_lib.pcnn_depth_blob_train_fwd
    assert g(buf, 1, buf, buf, None, 1, 8, 8, mean, None, buf, None) == -1
    assert b"NULL" in native_lib.pcnn_last_error()
    assert g(buf, 1, buf, buf, None, 1, -8, 8, mean, buf, buf, None) == -1
    assert b"bad shape" in native_lib.pcnn_last_error()
