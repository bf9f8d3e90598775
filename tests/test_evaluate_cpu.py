"""CPU side of the device evaluator (posecnn_b200/evaluate.py, DESIGN.md §14): the oracle tests/eval_ref.py against the goldens
made with the reference's own pose_error.py, the host helpers, and argument rejection by the C ABI before any CUDA work."""
import ctypes
import os

import numpy as np
import pytest

from posecnn_b200 import synth
from posecnn_b200.evaluate import LOV_EVAL_SYMMETRIC, gt_rows_from_meta
from tests import eval_ref

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "eval.npz"))


def case(tag):
    return {k[len(tag) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(tag + "_")}


@pytest.mark.parametrize("tag", eval_ref.CASES)
def test_oracle_matches_reference_scorer(tag):
    g = case(tag)
    c = eval_ref.make_case(tag)
    for k, v in c.items():                                   # the generator still makes the committed inputs
        np.testing.assert_array_equal(np.asarray(v), g[k], err_msg=k)
    C = int(g["C"])
    pts = synth.make_model_points(C, 2620)
    np.testing.assert_array_equal(eval_ref.fast_hist(g["gt_label"].reshape(-1), g["label"].reshape(-1), C), g["hist"])
    pairs, errors, flags, counts = eval_ref.score(g["gt_rows"], g["rois"], list(g["poses"]), int(g["num_rows"]), g["meta"], pts,
                                                  g["symmetric"], g["threshold"], g["flip_z"], C)
    np.testing.assert_array_equal(pairs, g["pairs"])
    np.testing.assert_allclose(errors, g["errors"], rtol=0, atol=1e-12)
    np.testing.assert_array_equal(flags, g["flags"])
    np.testing.assert_array_equal(counts, g["counts"])


def test_golden_cases_cover_the_edge_cases():
    lov, egg = case("lov"), case("egg")
    assert (lov["gt_label"] == -1).any() and (egg["gt_label"] == -1).any()
    assert not lov["poses"][1].reshape(-1, 7)[:, :4].any(axis=1).all()            # a zero quaternion
    j = lov["pairs"][:, 0]
    assert (np.bincount(j) > 1).any()                                               # duplicate detections of one gt
    fg = [i for i in range(lov["gt_rows"].shape[0]) if 0 < lov["gt_rows"][i, 1] < 22]
    assert set(fg) - set(j.tolist())                                                # a gt without a detection
    assert (lov["errors"][..., 0] < 1e-3).any()                                     # near-identity rotations
    assert set(lov["gt_rows"][:, 1].astype(int)) & {13, 16, 21}
    assert (egg["flags"] & 4).any() and not (egg["flags"] & 4).all()                # both sides of 90 degrees
    flipped = (egg["errors"][..., 0] > 90) == ((egg["flags"] & 4) > 0)
    assert flipped.all()
    assert (lov["counts"][:, 0].sum(1) == len(fg)).all()                           # count_all: once per gt and set


def test_summary_figures():
    g = case("lov")
    s = eval_ref.summary(g["hist"], g["counts"], ["poses", "poses_refined", "poses_icp"])
    hist = g["hist"].astype(np.float64)
    assert s["overall_accuracy"] == np.diag(hist).sum() / hist.sum()
    acc = s["poses"]["poses"]["accuracy"]
    a = g["counts"][0, 0]
    assert np.isnan(acc[a == 0]).all() and np.isfinite(acc[a > 0]).all()


def test_host_helpers():
    assert np.flatnonzero(LOV_EVAL_SYMMETRIC).tolist() == [13, 16, 21]
    assert np.flatnonzero(synth.LOV_SYMMETRY).tolist() == [16, 21]
    rng = np.random.default_rng(3)
    poses = rng.normal(size=(3, 4, 2))
    rows = gt_rows_from_meta(5, np.array([[3], [7]]), poses)
    assert rows.shape == (2, 14) and rows.dtype == np.float32
    assert rows[:, 0].tolist() == [5, 5] and rows[:, 1].tolist() == [3, 7]
    np.testing.assert_array_equal(rows[1, 2:].reshape(3, 4), poses[:, :, 1].astype(np.float32))
    one = gt_rows_from_meta(0, [4], poses[:, :, 0])                          # lov.py:572-573: a [3,4] pose is one object
    np.testing.assert_array_equal(one[0], np.r_[0, 4, rows[0, 2:]])
    with pytest.raises(ValueError):
        gt_rows_from_meta(0, [1, 2, 3], poses)
    thr = eval_ref.default_threshold(synth.extents_for(22))
    assert thr.dtype == np.float32 and thr[0] == 0 and thr[1] == np.float32(0.1 * np.linalg.norm(synth.extents_for(22)[1]))


def test_abi_argument_validation_without_gpu(native_lib):
    lib = native_lib
    p = ctypes.c_void_p(16)
    assert lib.pcnn_eval_confusion(p, p, 100, 1, p, p, None) == -1 and b"C = 1" in lib.pcnn_last_error()
    assert lib.pcnn_eval_confusion(p, p, 100, 129, p, p, None) == -1
    assert lib.pcnn_eval_confusion(None, p, 100, 22, p, p, None) == -1 and b"null" in lib.pcnn_last_error()
    assert lib.pcnn_eval_confusion(p, p, 100, 22, p, None, None) == -1
    assert lib.pcnn_eval_confusion(p, p, 0, 22, p, p, None) == 0                   # nothing to count: no launch
    args = lambda **kw: dict(dict(gt=p, num_gt=8, rois=p, stride=7, cap=64, num_rows=p, p0=p, p1=None, p2=None, p3=None, S=1, meta=p,
                                  num_meta=48, B=2, off=0, points=p, C=22, P=2620, sym=p, thr=p, flip=p, pairs=p, errors=p, flags=p,
                                  num_pairs=p, counts=p, status=p, stream=None), **kw)
    call = lambda a: lib.pcnn_eval_pose_errors(*a.values())
    assert call(args(num_gt=-1)) == -1 and b"num_gt" in lib.pcnn_last_error()
    assert call(args(num_gt=4097)) == -1
    assert call(args(stride=1)) == -1 and b"roi_stride" in lib.pcnn_last_error()
    assert call(args(S=0)) == -1 and b"num_sets" in lib.pcnn_last_error()
    assert call(args(S=5)) == -1
    assert call(args(S=2)) == -1 and b"pose set 1" in lib.pcnn_last_error()
    assert call(args(C=1)) == -1 and b"C = 1" in lib.pcnn_last_error()
    assert call(args(P=0)) == -1 and call(args(P=4097)) == -1
    assert call(args(num_meta=8)) == -1 and b"num_meta" in lib.pcnn_last_error()
    assert call(args(B=0)) == -1
    assert call(args(points=None)) == -1 and b"null input" in lib.pcnn_last_error()
    assert call(args(flip=None)) == -1
    assert call(args(errors=None)) == -1 and b"null output" in lib.pcnn_last_error()
    assert call(args(status=None)) == -1
    assert call(args(num_gt=4096, cap=1 << 20)) == -1 and b"pairs" in lib.pcnn_last_error()
    assert lib.pcnn_eval_gt_rows_from_blob(p, -1, p, None) == -1
    assert lib.pcnn_eval_gt_rows_from_blob(None, 3, p, None) == -1 and b"null" in lib.pcnn_last_error()
    assert lib.pcnn_eval_gt_rows_from_blob(None, 0, None, None) == 0
