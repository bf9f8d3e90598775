"""GPU parity of Houghvotinggpu (hand-written sm_90a kernels, through the C ABI) against the
CPU oracle.  Tolerances: integer outputs exact; box / pose 1e-4 (SURVEY.md §8(c))."""
import numpy as np
import pytest
import torch

from oracle import oracle
from posecnn_b200 import synth
from tests.util import assert_hough_rows_equal, to_np

pytestmark = pytest.mark.gpu


def _dev(sc, dev):
    t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    gt = t(sc["gt"]) if sc["gt"] is not None and len(sc["gt"]) else None
    return t(sc["label"]), t(sc["vertex"]), t(sc["extents"]), t(sc["meta"]), gt


def _check_planes(got, dbg, max_bad_frac=0.0):
    votes, amb = dbg["votes"], dbg["ambig"]
    diff = np.abs(to_np(got) - votes)
    bad = diff > amb
    assert bad.mean() <= max_bad_frac, f"{bad.sum()} cells differ beyond the ambiguity bound; max diff {diff.max()}"
    return int((diff > 0).sum()), int(amb.sum())


@pytest.mark.parametrize("seed,noise,skip", [(3, 0.05, 10), (4, 0.0, 10), (5, 0.2, 3), (6, 0.05, 1)])
def test_vote_planes_match_oracle_small(cuda, seed, noise, skip):
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    sc = synth.make_scene(batch=2, height=120, width=160, num_classes=5, objects_per_image=3, seed=seed,
                          dir_noise=noise, min_pixels=520)
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], sc["gt"], 0, -1.0, 0.02, skip,
                                     debug=True)
    lab, vert, ext, meta, gt = _dev(sc, cuda)
    planes = op.hough_vote_planes(lab, vert, ext, meta, skip)
    assert dbg["votes"].max() > 10
    _check_planes(planes, dbg)


@pytest.mark.parametrize("is_train", [0, 1])
@pytest.mark.parametrize("seed", [3, 7, 9])
def test_outputs_match_oracle_small(cuda, seed, is_train):
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    sc = synth.make_scene(batch=3, height=120, width=160, num_classes=6, objects_per_image=3, seed=seed, min_pixels=520)
    want = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], sc["gt"], is_train, -1.0, 0.02, 10)
    lab, vert, ext, meta, gt = _dev(sc, cuda)
    got = op.hough_voting_gpu(lab, vert, ext, meta, gt, is_train, -1.0, 0.02, 10)
    assert_hough_rows_equal(got, want, is_train)
    box, pose, target, weight, domain, nr, status = op.hough_voting_gpu_capacity(lab, vert, ext, meta, gt, is_train, -1.0,
                                                                                 0.02, 10)
    assert to_np(status)[1] == 0, "interval-scan votes differ from the per-cell recount at a selected maximum"
    assert not to_np(box)[int(nr.item()):].any()          # capacity rows beyond num_rois stay zero


def test_threshold_mode_matches_oracle(cuda):
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    sc = synth.make_scene(batch=2, height=120, width=160, num_classes=5, objects_per_image=3, seed=13, min_pixels=520,
                          dir_noise=0.1)
    for vote_thr, per_thr in [(20.0, 0.0), (30.0, 0.002), (5.0, 0.02)]:
        want = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], sc["gt"], 0, vote_thr, per_thr, 10)
        lab, vert, ext, meta, gt = _dev(sc, cuda)
        got = op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, vote_thr, per_thr, 10)
        assert_hough_rows_equal(got, want, 0)


def test_edge_cases(cuda):
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    # (a) nothing above the 500-pixel label threshold -> one all-zero dummy row
    sc = synth.make_scene(batch=2, height=60, width=80, num_classes=3, objects_per_image=1, seed=2, min_pixels=100)
    lab, vert, ext, meta, gt = _dev(sc, cuda)
    got = op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10)
    assert got[0].shape == (1, 7) and not to_np(got[0]).any() and got[4].shape == (1,)
    # (b) all-background labels, labels outside [0, C), NaN / inf / huge vertex values must not crash or hang
    sc = synth.make_scene(batch=1, height=120, width=160, num_classes=4, objects_per_image=2, seed=3, min_pixels=520)
    v = sc["vertex"].copy()
    v[0, ::7, ::5, :] = np.nan
    v[0, 1::7, ::5, :] = np.inf
    v[0, 2::7, ::5, :] = -1e30
    l = sc["label"].copy()
    l[0, :3, :3] = 99
    l[0, 3:5, :3] = -5
    sc2 = dict(sc, vertex=v, label=l)
    want = oracle.hough_voting_gpu(l, v, sc["extents"], sc["meta"], sc["gt"], 0, -1.0, 0.02, 10)
    lab, vert, ext, meta, gt = _dev(sc2, cuda)
    got = op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10)
    assert_hough_rows_equal(got, want, 0)
    # (c) ROI cap 128 / B: batch 64 keeps 2 maxima per image (SURVEY finding 3)
    sc = synth.make_scene(batch=1, height=120, width=160, num_classes=6, objects_per_image=4, seed=5, min_pixels=520)
    rep = lambda a: np.repeat(a, 64, 0)
    lab, vert, ext, meta, gt = _dev(dict(sc, label=rep(sc["label"]), vertex=rep(sc["vertex"]), meta=rep(sc["meta"])), cuda)
    got = op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10)
    assert got[0].shape[0] == 128
    b = to_np(got[0])
    np.testing.assert_array_equal(np.bincount(b[:, 0].astype(int)), [2] * 64)
    np.testing.assert_array_equal(b[:2, 1:], b[126:, 1:])      # identical images -> identical rows
    # (d) ragged sizes: width not a multiple of 32, height not a multiple of the 32-row band
    sc = synth.make_scene(batch=2, height=101, width=147, num_classes=4, objects_per_image=2, seed=21, min_pixels=520)
    want, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], sc["gt"], 0, -1.0, 0.02, 10,
                                        debug=True)
    lab, vert, ext, meta, gt = _dev(sc, cuda)
    _check_planes(op.hough_vote_planes(lab, vert, ext, meta, 10), dbg)
    assert_hough_rows_equal(op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10), want, 0)
    # (e) gradient op: zeros of the right shapes
    gl, gv = op.hough_voting_gpu_grad(lab, vert, got[0])
    assert gl.shape == lab.shape and gl.dtype == torch.float32 and not gl.any() and gv.shape == vert.shape and not gv.any()


def test_full_size_frame_matches_oracle(cuda):
    """configs[1]: one 640x480 frame, 22 classes (C oracle takes a few seconds with OpenMP)."""
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    sc = synth.make_scene(batch=1, height=480, width=640, num_classes=22, seed=1234)
    want, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], sc["gt"], 0, -1.0, 0.02, 10,
                                        debug=True)
    lab, vert, ext, meta, gt = _dev(sc, cuda)
    ndiff, namb = _check_planes(op.hough_vote_planes(lab, vert, ext, meta, 10), dbg)
    got = op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10)
    assert want[0].shape[0] >= 3
    assert_hough_rows_equal(got, want, 0)
    print(f"full frame: {ndiff} cells differ (all within ambiguity), {namb} ambiguous pairs")


def test_batch32_properties(cuda):
    """BASELINE batch 32 at full size: size-independent properties instead of the (slow) oracle —
    batch invariance (image i of a batch == the same image alone, up to the 128/B cap) and
    determinism (two runs bit-identical)."""
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    sc = synth.make_scene(batch=32, height=480, width=640, num_classes=22, seed=4321)
    lab, vert, ext, meta, gt = _dev(sc, cuda)
    a = [to_np(x) for x in op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10)]
    b = [to_np(x) for x in op.hough_voting_gpu(lab, vert, ext, meta, gt, 0, -1.0, 0.02, 10)]
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    assert np.bincount(a[0][:, 0].astype(int), minlength=32).max() <= 4          # cap = 128 / 32
    for i in (0, 13, 31):
        single = [to_np(x) for x in op.hough_voting_gpu(lab[i:i + 1], vert[i:i + 1], ext, meta[i:i + 1], None, 0, -1.0,
                                                        0.02, 10)]
        rows = a[0][a[0][:, 0] == i]
        k = rows.shape[0]
        assert k == min(4, single[0].shape[0])
        np.testing.assert_array_equal(rows[:, 1:], single[0][:k, 1:])
        np.testing.assert_array_equal(a[1][a[0][:, 0] == i], single[1][:k])
