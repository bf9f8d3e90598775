"""Object-coordinate pose estimation (DESIGN.md §13) without a GPU: the float64 restatement tests/coord_pose_ref.py recovers the
planted poses of analytic scenes, its Kabsch / Rodrigues helpers agree with closed forms, and the C ABI rejects bad arguments."""
import ctypes
import os

import numpy as np
import pytest

from posecnn_b200 import synth
from tests import coord_pose_ref as ref

PLANTED_ROT_DEG, PLANTED_TRANS_M = 0.5, 0.002     # noise-free scenes


def rot_err_deg(Ra, Rb):
    return float(np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1))))


def run_oracle(sc, b, key, C):
    cam = (sc["meta"][b, 0], sc["meta"][b, 4], sc["meta"][b, 2], sc["meta"][b, 5])
    return ref.estimate_image(sc["label"][b], sc["depth"][b], sc["vertex"][b], sc["extents"], cam, 10000.0, key, C)


def test_oracle_recovers_planted_poses():
    C = 6
    sc = synth.make_coordinate_scene(batch=1, num_classes=C, objects_per_image=2, seed=3)
    out = run_oracle(sc, 0, 12345, C)
    checked = 0
    for row in sc["poses"]:
        c = int(row[1])
        if (sc["label"][0] == c).sum() <= ref.MIN_AREA:
            continue
        R, t = synth.quat_to_rot(row[2:6]), row[6:9]
        assert rot_err_deg(out["poses"][c, :, :3], R) < PLANTED_ROT_DEG
        assert np.linalg.norm(out["poses"][c, :, 3] - t) < PLANTED_TRANS_M
        assert out["info"][c, 2] > ref.MIN_FINAL
        checked += 1
    assert checked >= 1
    # every other class: no pose
    for c in range(C):
        if c not in {int(r[1]) for r in sc["poses"]}:
            assert not out["poses"][c].any()


def test_subset_rule_takes_every_pixel_at_rate_one_and_skips_holes():
    L = np.arange(900, dtype=np.int64)
    L[5] |= ref.HOLE
    pos = ref.subset(L, 1, 0, 7)            # 1000 / 900 >= 1: every pixel but the hole
    assert len(pos) == 899 and 5 not in pos
    L = np.arange(20000, dtype=np.int64)
    pos = ref.subset(L, 1, 0, 7)            # rate 0.05
    assert 0.6 * 1000 < len(pos) < 1.4 * 1000 and np.all(np.diff(pos) >= 1)


def test_kabsch_and_rodrigues_closed_forms():
    rng = np.random.default_rng(0)
    R = synth.quat_to_rot(synth._rand_quat(rng))
    t = rng.normal(size=3)
    A = rng.normal(size=(5, 3))
    Rk, tk = ref.kabsch(A, A @ R.T + t)
    np.testing.assert_allclose(Rk, R, atol=1e-12)
    np.testing.assert_allclose(tk, t, atol=1e-12)
    assert ref.kabsch(np.outer(np.arange(3.0), [1, 2, 3]), np.outer(np.arange(3.0), [1, 2, 3])) is None   # collinear
    np.testing.assert_allclose(ref.rodrigues_exp(ref.rodrigues_log(R)), R, atol=1e-12)


def test_abi_argument_validation_without_gpu(native_lib):
    nbytes = ctypes.c_size_t(0)
    lib = native_lib
    lib.pcnn_last_error.restype = ctypes.c_char_p
    assert lib.pcnn_coord_pose3d_workspace_bytes(2, 480, 640, 22, ctypes.byref(nbytes)) == 0 and nbytes.value > 0
    assert lib.pcnn_coord_pose3d_workspace_bytes(2, 480, 640, 1, ctypes.byref(nbytes)) == -1
    assert b"C = 1" in lib.pcnn_last_error()
    assert lib.pcnn_coord_pose3d_workspace_bytes(2, 480, 640, 129, ctypes.byref(nbytes)) == -1
    assert lib.pcnn_coord_pose3d_workspace_bytes(2, 480, 640, 22, None) == -1
    p = ctypes.c_void_p(16)
    args = lambda **kw: dict(dict(label=p, vertex=p, lowres=None, bias=None, depth=p, meta=p, num_meta=48, ext=p, keys=p, B=1, H=480,
                                  W=640, C=22, factor=ctypes.c_float(10000.0), poses=p, info=p, th=None, tr=None, ws=p,
                                  nbytes=ctypes.c_size_t(1 << 40), stream=None), **kw)
    call = lambda a: lib.pcnn_coord_pose3d_fwd(*a.values())
    assert call(args(label=None)) == -1
    assert call(args(vertex=None)) == -1 and b"lowres" in lib.pcnn_last_error()
    assert call(args(vertex=None, lowres=p, bias=p, H=481)) == -1 and b"multiples of 8" in lib.pcnn_last_error()
    assert call(args(num_meta=5)) == -1
    assert call(args(factor=ctypes.c_float(0.0))) == -1
    assert call(args(nbytes=ctypes.c_size_t(16))) == -1 and b"workspace" in lib.pcnn_last_error()


def golden_record_cases():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "coord_pose_records.npz"))
    n = sum(1 for k in g.files if k.startswith("rois_"))
    return g["K"], [(g[f"poses_tmp_{i}"], float(g[f"im_scale_{i}"]), g[f"rois_{i}"], g[f"poses_{i}"]) for i in range(n)]


def test_record_assembly_equals_the_reference():
    """The restated record assembly against the reference's own lines (tests/golden/make_golden_coord_pose.py)."""
    K, cases = golden_record_cases()
    for P, scale, rois, poses in cases:
        C = P.shape[2]
        r, p = ref.records(P.transpose(2, 0, 1), synth.extents_for(C), K, scale)
        assert r.shape == rois.shape
        np.testing.assert_array_equal(r[:, :2], rois[:, :2])
        np.testing.assert_allclose(r[:, 2:], rois[:, 2:], rtol=1e-6, atol=1e-3)
        np.testing.assert_allclose(p, poses, rtol=0, atol=1e-6)
