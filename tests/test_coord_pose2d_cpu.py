"""Colour-only object-coordinate pose estimation (DESIGN.md §13) without a GPU: the float64 restatement tests/coord_pose2d_ref.py
recovers the planted poses of analytic scenes, its P3P agrees with OpenCV's, its subset rule is the depth estimator's on hole-free
lists, and the C ABI rejects bad arguments."""
import ctypes

import numpy as np
import pytest

from posecnn_b200 import synth
from tests import coord_pose2d_ref as ref2
from tests import coord_pose_ref as ref
from tests.test_coord_pose_cpu import PLANTED_ROT_DEG, PLANTED_TRANS_M, rot_err_deg


def cam_of(sc, b):
    return (sc["meta"][b, 0], sc["meta"][b, 4], sc["meta"][b, 2], sc["meta"][b, 5])


def test_oracle_recovers_planted_poses():
    C = 6
    sc = synth.make_coordinate_scene(batch=1, num_classes=C, objects_per_image=2, seed=3)
    out = ref2.estimate_image(sc["label"][0], sc["vertex"][0], sc["extents"], cam_of(sc, 0), 12345, C)
    checked = 0
    for row in sc["poses"]:
        c = int(row[1])
        if (sc["label"][0] == c).sum() <= ref.MIN_AREA:
            continue
        R, t = synth.quat_to_rot(row[2:6]), row[6:9]
        assert rot_err_deg(out["poses"][c, :, :3], R) < PLANTED_ROT_DEG
        assert np.linalg.norm(out["poses"][c, :, 3] - t) < PLANTED_TRANS_M
        assert out["info"][c, 3] == -1 and out["info"][c, 2] > 0
        checked += 1
    assert checked >= 1
    for c in range(C):
        if c not in {int(r[1]) for r in sc["poses"]}:
            assert not out["poses"][c].any()


def test_p3p_agrees_with_opencv():
    """Random four-point sets in front of the camera: the oracle's pose against cv2.solvePnP(SOLVEPNP_P3P).  A disagreement is
    allowed only where two roots reproject the fourth point almost equally well (a near-tie of the selection)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    fx, fy, px, py = 572.4114, 573.57043, 325.2611, 242.04899
    K = np.array([[fx, 0, px], [0, fy, py], [0, 0, 1]], np.float32)
    agree = ties = 0
    for _ in range(200):
        obj = rng.uniform(-0.1, 0.1, (4, 3)).astype(np.float32)
        R = synth.quat_to_rot(synth._rand_quat(rng))
        t = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.5, 1.5)])
        cam = obj.astype(np.float64) @ R.T + t
        uv = (cam[:, :2] / cam[:, 2:]) * [fx, fy] + [px, py]
        uv = np.round(uv).astype(np.float32)                 # integer pixels, as the estimator samples them
        sol = ref2.p3p(obj, uv[:, 0], uv[:, 1], tuple(float(x) for x in (fx, fy, px, py)))
        ok, rvec, tvec = cv2.solvePnP(obj, uv, K, None, flags=cv2.SOLVEPNP_P3P)
        if sol is None or not ok:          # no real root on one side: counted as a disagreement
            continue
        Rc = cv2.Rodrigues(rvec)[0]
        if rot_err_deg(sol[0], Rc) < 1e-3 and np.linalg.norm(sol[1] - tvec[:, 0]) < 1e-5:
            agree += 1
            continue
        # near-tie: both poses reproject the fourth point within a pixel of each other
        e_ref = np.hypot(*(np.array(ref2.project(*sol, (fx, fy, px, py), obj[3])) - uv[3]))
        e_cv = np.hypot(*(np.array(ref2.project(Rc, tvec[:, 0], (fx, fy, px, py), obj[3])) - uv[3]))
        assert abs(e_ref - e_cv) < 1.0, (e_ref, e_cv)
        ties += 1
    print(f"\n[p3p vs OpenCV] {agree} agree, {ties} near-ties")
    assert agree >= 150


def test_p3p_exact_on_noise_free_points():
    rng = np.random.default_rng(3)
    cam = (600.0, 600.0, 320.0, 240.0)
    for _ in range(50):
        obj = rng.uniform(-0.1, 0.1, (4, 3)).astype(np.float32)
        R = synth.quat_to_rot(synth._rand_quat(rng))
        t = np.array([0.0, 0.0, 1.0]) + rng.uniform(-0.1, 0.1, 3)
        q = obj.astype(np.float64) @ R.T + t
        u, v = q[:, 0] / q[:, 2] * 600 + 320, q[:, 1] / q[:, 2] * 600 + 240
        Rs, ts = ref2.p3p(obj, u, v, cam)
        assert rot_err_deg(Rs, R) < 1e-5 and np.linalg.norm(ts - t) < 1e-7     # arccos resolves ~1e-6 deg


def test_quartic_roots():
    for roots in ([-2.0, 0.5, 1.0, 3.0], [0.9, 1.1], [1.0, 1.0 + 1e-6, 2.0, 5.0]):
        poly = np.poly(roots + ([complex(0.3, 1.0), complex(0.3, -1.0)] if len(roots) == 2 else [])).real
        got = ref2.quartic_roots(list(poly[1:]))
        np.testing.assert_allclose(got, sorted(roots), rtol=0, atol=1e-9)


def test_subset_rule_is_the_depth_estimators_on_hole_free_lists():
    sc = synth.make_coordinate_scene(batch=1, num_classes=6, objects_per_image=2, seed=4)
    lists = ref.pixel_lists(sc["label"][0], np.ones_like(sc["depth"][0]), 6)
    lists_d = ref.pixel_lists(sc["label"][0], sc["depth"][0], 6)
    for c in range(1, 6):
        if len(lists[c]) <= ref.MIN_AREA:
            continue
        assert not np.any(lists[c] & ref.HOLE)
        for r in range(ref.ROUNDS):
            np.testing.assert_array_equal(ref.subset(lists[c], c, r, 99), ref.subset(lists[c] | 0, c, r, 99))
            if not np.any(lists_d[c] & ref.HOLE):       # the scene's depth has no hole on this object: the same positions
                np.testing.assert_array_equal(ref.subset(lists[c], c, r, 99), ref.subset(lists_d[c], c, r, 99))


def test_counter_spaces_are_disjoint():
    h, att = 255, 1023
    spaces = {ref.ctr_hyp(h, att) >> 60, ref.ctr_sub(21, 7, 5) >> 60, ref.ctr_fil(h, 8, 999) >> 60, ref2.ctr_p2a(h, att) >> 60,
              ref2.ctr_p2b(h, att) >> 60}
    assert spaces == {1, 2, 3, 4, 5}


def test_abi_argument_validation_without_gpu(native_lib):
    nbytes = ctypes.c_size_t(0)
    lib = native_lib
    assert lib.pcnn_coord_pose2d_workspace_bytes(2, 480, 640, 22, ctypes.byref(nbytes)) == 0 and nbytes.value > 0
    n3 = ctypes.c_size_t(0)
    assert lib.pcnn_coord_pose3d_workspace_bytes(2, 480, 640, 22, ctypes.byref(n3)) == 0 and n3.value == nbytes.value
    assert lib.pcnn_coord_pose2d_workspace_bytes(2, 480, 640, 1, ctypes.byref(nbytes)) == -1
    assert b"C = 1" in lib.pcnn_last_error()
    assert lib.pcnn_coord_pose2d_workspace_bytes(2, 480, 640, 129, ctypes.byref(nbytes)) == -1
    assert lib.pcnn_coord_pose2d_workspace_bytes(0, 480, 640, 22, ctypes.byref(nbytes)) == -1
    assert lib.pcnn_coord_pose2d_workspace_bytes(2, 480, 640, 22, None) == -1
    p = ctypes.c_void_p(16)
    args = lambda **kw: dict(dict(label=p, vertex=p, lowres=None, bias=None, meta=p, num_meta=48, ext=p, keys=p, B=1, H=480, W=640, C=22,
                                  poses=p, info=p, th=None, tr=None, ws=p, nbytes=1 << 40, stream=None), **kw)
    call = lambda a: lib.pcnn_coord_pose2d_fwd(*a.values())
    assert call(args(label=None)) == -1 and b"coord_pose2d" in lib.pcnn_last_error()
    assert call(args(keys=None)) == -1
    assert call(args(vertex=None)) == -1 and b"lowres" in lib.pcnn_last_error()
    assert call(args(vertex=None, lowres=p, bias=p, H=481)) == -1 and b"multiples of 8" in lib.pcnn_last_error()
    assert call(args(num_meta=5)) == -1
    assert call(args(C=129)) == -1
    assert call(args(nbytes=16)) == -1 and b"workspace" in lib.pcnn_last_error()
