"""CPU checks of the detection records (DESIGN.md §16): the NumPy restatement tests/det_post_ref.py against the reference's own
post-processing (tests/golden/det_post.npz, tests/golden/make_golden_det_post.py), the canonical tie rule, and the argument
checks of pcnn_det_records_fwd, which reject bad input before any CUDA work.

Selection and boxes must equal the reference exactly.  The depth z of each search must be bit-equal wherever the two searches
evaluate the same points; the reference's objective sums RT @ x3d with BLAS sgemm (its own order, with FMA) where the
restatement follows the device's order, so a comparison whose two values lie within the objective's fp32 sensitivity
(det_post_ref.sensitivity) may be decided the other way.  Every other search is replayed on the reference's own objective
values (det_post_ref.replay): it must then evaluate exactly the reference's points and end at its z, and each decision the
two sets of values take differently must have its margin within the sensitivity.  Those cases are counted and printed.
"""
import ctypes
import math
import os

import numpy as np
import pytest

from tests import det_post_ref as ref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "det_post.npz"))
TAGS = ("lov", "linemod")


def case(tag):
    return {k[len(tag) + 1:]: GOLD[k] for k in GOLD.files if k.startswith(tag + "_")}


def compare_with_golden(tag, dets, poses, trace, only=None):
    """dets / poses / trace: the filled slots (classes ascending per image) of a run on the golden inputs; only: the records
    whose translation is checked (default all).  Returns the number of searches whose decisions differ (all explained)."""
    g = case(tag)
    np.testing.assert_array_equal(dets[:, :2], g["ref_dets"][:, :2])              # image and class
    np.testing.assert_array_equal(dets[:, 6], g["ref_dets"][:, 6])                # score
    np.testing.assert_array_equal(poses[:, :4], g["ref_poses"][:, :4])            # the raw quaternion
    points = g["points"]
    explained = 0
    for i in (range(dets.shape[0]) if only is None else only):
        b, j = int(dets[i, 0]), int(dets[i, 1])
        K = g["meta"][b, :9].astype(np.float64).reshape(3, 3)
        n = int(g["ref_evals"][i])
        want_xs, want_z = g["ref_xs"][i, :n], float(g["ref_z"][i])
        s = ref.translation(dets[i, 2:6], poses[i, :4], points[j], K)[1]
        if np.array_equal(np.asarray(s.xs), want_xs):                            # the same decisions: bit-equal
            assert s.z == want_z and (s.nit, s.nfev) == tuple(g["ref_nit_nfev"][i]), i
            np.testing.assert_array_equal(poses[i, 4:], g["ref_poses"][i, 4:])
            if trace is not None:
                assert tuple(trace[i]) == (s.nit, s.nfev)
            continue
        r, flipped = ref.replay(dets[i, 2:6], poses[i, :4], points[j], K, want_xs, g["ref_fs"][i, :n])
        assert np.array_equal(np.asarray(r.xs), want_xs) and r.z == want_z, i     # the same algorithm on the same values
        assert (r.nit, r.nfev) == tuple(g["ref_nit_nfev"][i]), i
        assert flipped and all(m <= tol for _, m, tol in flipped), (i, flipped)
        explained += 1
        print(f"{tag} record {i} (image {b}, class {j}): {len(flipped)} decisions taken the other way, margin <= fp32 "
              f"sensitivity: {[(k, f'{m:.3g} <= {tol:.3g}') for k, m, tol in flipped]}")
    return explained


@pytest.mark.parametrize("tag", TAGS)
def test_restatement_equals_reference(tag):
    g = case(tag)
    dets, poses, num, trace, boxes = ref.records(g["cls_prob"], g["bbox_pred"], g["poses_tanh"], g["rois"], g["num_rois"],
                                                 g["im_hw"], g["meta"], g["points"])
    filled = dets[:, 1] > 0
    assert int(num.sum()) == filled.sum() == g["ref_dets"].shape[0]
    np.testing.assert_array_equal(dets[filled, 2:6], g["ref_dets"][:, 2:6])       # boxes exactly (numpy's exp on both sides)
    assert (dets[~filled, 1:] == 0).all() and (poses[~filled] == 0).all()
    n = compare_with_golden(tag, dets[filled], poses[filled], trace[filled])
    print(f"{tag}: {filled.sum()} records, {n} searches explained by decisions within the fp32 sensitivity")


def test_golden_covers_the_cases():
    lov, lm = case("lov"), case("linemod")
    for g, C in ((lov, 22), (lm, 2)):
        assert g["cls_prob"].shape[1] == C
        d = g["ref_dets"]
        assert (d[:, 4] - d[:, 2] == 0).any()                                    # clipped to zero width
        assert ((d[:, 2] == 0) & (d[:, 3] == 0) & (d[:, 4] == 639) & (d[:, 5] == 479)).any()   # the full image
        assert (g["ref_poses"][:, :4] == 0).all(1).any()                          # a zero quaternion
        assert g["ref_z"].max() > 100                                             # a tiny box: large depth
        B = g["num_rois"].shape[0]
        assert len({(int(b), int(c)) for b, c in d[:, :2]}) < B * (C - 1)         # a class with nothing above 0.02
    assert (np.concatenate([lov["ref_nit_nfev"][:, 1], lm["ref_nit_nfev"][:, 1]]) == 200).any()   # the evaluation cap


def test_ties_go_to_the_lowest_row():
    """cls_score's ReLU makes rows with all logits <= 0 exactly 1/C in every class: the canonical winner is the lowest row."""
    s = np.full((6, 3), np.float32(1 / 3), np.float32)
    s[0, 1] = np.float32(0.2)
    s[4, 2] = np.float32(0.9)
    s[5, 2] = np.float32(0.9)
    assert ref.select(s, 6) == [(1, 1), (2, 4)]
    assert ref.select(s, 5) == [(1, 1), (2, 4)]
    s[:, 1] = np.float32(0.02)                                                   # not above the threshold
    s[2, 2] = np.float32(np.nan)                                                 # NaN is never selected
    assert ref.select(s, 4) == [(2, 0)]
    assert ref.select(s, 0) == []


@pytest.mark.parametrize("f", [lambda z: (z - 1.7) ** 2, lambda z: -z, lambda z: math.nan if z > 0.6 else (z - 2.0) ** 2,
                               lambda z: 0.0 if z > 3 else 1.0 / z, lambda z: math.inf if z < 0.52 else z])
def test_search_steps_like_scipy(f):
    """The restated search and scipy's minimize evaluate the same points and stop alike (a smooth minimum, an unbounded
    descent to the evaluation cap, NaN, a flat region, inf)."""
    from scipy.optimize import minimize
    seen = []
    r = minimize(lambda x: seen.append(float(x[0])) or f(float(x[0])), 0.5, method="nelder-mead")
    s = ref.Search(lambda z: ref.Value(f(z))).run()
    assert s.xs == seen and s.z == float(r.x[0]) and (s.nit, s.nfev) == (r.nit, r.nfev)


def test_entry_point_rejects_bad_arguments(native_lib):
    buf = ctypes.create_string_buffer(256)
    err = lambda: native_lib.pcnn_last_error()

    def call(B=1, rows=300, C=22, im_h=480, im_w=640, num_meta=48, P=2620, null=None):
        p = [buf] * 11
        if null is not None:
            p[null] = None
        return native_lib.pcnn_det_records_fwd(p[0], p[1], p[2], p[3], p[4], B, rows, C, im_h, im_w, p[5], num_meta, p[6], P, p[7],
                                               p[8], p[9], p[10], None)
    assert call(C=1) == -1 and b"C = 1" in err()
    assert call(C=129) == -1 and b"C = 129" in err()
    assert call(P=0) == -1 and b"P = 0" in err()
    assert call(P=4097) == -1 and b"P = 4097" in err()
    assert call(B=0) == -1 and b"B = 0" in err()
    assert call(B=65536) == -1
    assert call(rows=0) == -1 and b"rows" in err()
    assert call(im_w=0) == -1 and b"image size" in err()
    assert call(num_meta=8) == -1 and b"num_meta" in err()
    for k in range(11):
        assert call(null=k) == -1 and b"NULL" in err()
