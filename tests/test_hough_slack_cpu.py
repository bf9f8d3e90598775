"""CPU tests of the oracle's exactness analysis of the Hough interval scan (oracle.hough_voting_gpu(..., slack=True),
DESIGN.md §3.3) and of the reference behaviour the device op must reproduce for directions whose norm underflows."""
import numpy as np
import pytest

from oracle import oracle
from tests import hough_ref as HR


def test_row_exact_hand_built():
    T, F = 1, 0
    # off the pixel's own row: empty or one interval
    assert oracle.hough_row_exact([F] * 7, 3, 5, False)
    assert oracle.hough_row_exact([F, T, T, T, F, F, F], 3, 5, False)
    assert oracle.hough_row_exact([T] * 7, 3, 5, False)
    assert oracle.hough_row_exact([F, F, F, F, F, F, T], 3, 5, False)
    assert not oracle.hough_row_exact([T, T, F, T, F, F, F], 3, 5, False)          # a hole
    assert not oracle.hough_row_exact([T, F, F, F, F, F, T], 3, 5, False)          # two intervals
    # the own row (x = 5, window 3 .. 9): empty or exactly one whole side
    assert oracle.hough_row_exact([F] * 7, 3, 5, True)
    assert oracle.hough_row_exact([F, F, F, T, T, T, T], 3, 5, True)               # x+1 .. wmax
    assert oracle.hough_row_exact([T, T, F, F, F, F, F], 3, 5, True)               # wmin .. x-1
    assert not oracle.hough_row_exact([F, F, F, F, T, T, T], 3, 5, True)           # x+2 .. wmax: dx = 1 fails
    assert not oracle.hough_row_exact([F, F, F, T, T, T, F], 3, 5, True)           # the last cell fails
    assert not oracle.hough_row_exact([F, T, F, F, F, F, F], 3, 5, True)           # x-1 only, x-2 fails
    assert oracle.hough_row_exact([F, F, F], 0, 2, True)                           # window clipped at the right border
    assert oracle.hough_row_exact([T, T, F], 0, 2, True)


def _tiny_dir_scene(scale, zero_components=True):
    """Class 2's directions scaled by `scale`; with zero_components, every 7th has u = 0 and some others v = 0."""
    sc = HR.blank_scene(1, 48, 64, 3, seed=5)
    HR.plant(sc, 0, 1, 20, 24, 14, 12, 0.8)
    ys, xs = HR.plant(sc, 0, 2, 46, 22, 14, 14, 0.7)
    sc["vertex"][0, ys, xs, 6:8] *= np.float32(scale)
    if zero_components:
        sc["vertex"][0, ys[::7], xs[::7], 6] = 0.0                                  # u = 0: whole rows on v's side
        sc["vertex"][0, ys[3::14], xs[3::14], 7] = 0.0                              # v = 0
    return sc


def _underflow_scene():
    return _tiny_dir_scene(1e-24)


def test_oracle_votes_half_plane_when_norm_underflows():
    """u*u + v*v underflows to n1 = 0 for every pixel of class 2: the reference's cosine dot / (n1 n2) is +-inf, so each
    sample votes for every cell of its window with dot > 0.  The oracle must show exactly that, with no irregular pair."""
    sc = _underflow_scene()
    skip = 1
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], None, 0, -1.0, 0.02, skip, slack=True)
    lab, vert = sc["label"][0], sc["vertex"][0]
    ys, xs = np.nonzero(lab == 2)
    u, v = vert[ys, xs, 6], vert[ys, xs, 7]
    assert ((u * u + v * v) == 0).all() and ((u != 0) | (v != 0)).all()
    H, W = lab.shape
    want = np.zeros((H, W), np.int64)
    cy, cx = np.mgrid[0:H, 0:W]
    d = np.exp(vert[ys, xs, 8])
    for k in range(xs.size):
        thr = oracle.project_box(sc["extents"], sc["meta"][0], 2, d[k])
        dx, dy = cx - xs[k], cy - ys[k]
        dot = np.float64(u[k]) * dx + np.float64(v[k]) * dy      # exact: u, v are tiny, their products with dx, dy exact
        want += (dot > 0) & (np.abs(dx) < thr) & (np.abs(dy) < thr)
    np.testing.assert_array_equal(dbg["votes"][0, 2], want)
    assert want.max() > 100 and (want > 0).sum() > 500
    assert dbg["pairs"][0, 2, 1] == 0 and dbg["pairs"][0, 2, 0] > 1000
    assert not dbg["slack"][0, 2].any()


def test_slack_marks_irregular_own_rows():
    """Pixels whose u / n1 is a few ulps from float32(0.9): on their own row the reference's cosine RN(RN(u dx) / RN(n1 |dx|))
    crosses the threshold at some dx and not others.  Where numpy predicts an own row that is not empty and not one whole
    side, the oracle must count an irregular pair and spread its slack over the window row; everything else stays exact."""
    sc = HR.blank_scene(1, 40, 96, 2, seed=9)
    ys, xs = HR.plant(sc, 0, 1, 48, 20, 40, 16, 0.1)
    dirs = HR.near_threshold_dirs()
    k = np.arange(dirs.shape[0]) * max(1, xs.size // dirs.shape[0])
    sc["vertex"][0, ys[k], xs[k], 3] = dirs[:, 0]
    sc["vertex"][0, ys[k], xs[k], 4] = dirs[:, 1]
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], None, 0, -1.0, 0.02, 1, slack=True)
    W = sc["label"].shape[2]
    irregular_rows = 0
    for (u, v), y, x in zip(dirs, ys[k], xs[k]):
        n1 = HR.norm_f32(u, v)
        dx = np.arange(-x, W - x).astype(np.float32)
        with np.errstate(invalid="ignore", divide="ignore"):
            c = (np.float32(u) * dx).astype(np.float32) / (n1 * np.abs(dx)).astype(np.float32)
        passes = c > np.float32(0.9)
        right, left = passes[dx > 0], passes[dx < 0]
        whole = (passes.sum() == 0) or (right.all() and not left.any()) or (left.all() and not right.any())
        if not whole:
            irregular_rows += 1
            assert dbg["slack"][0, 1, y].min() >= 1, (u, v, x, y)
    print(f"{dirs.shape[0]} near-threshold samples: {irregular_rows} irregular own rows (window = whole image width); "
          f"oracle: {int(dbg['pairs'][0, 1, 1])} irregular of {int(dbg['pairs'][0, 1, 0])} pairs")
    assert irregular_rows > 0
    assert dbg["pairs"][0, 1, 1] == irregular_rows          # the other rows of these samples are regular


@pytest.mark.parametrize("scale", [1e-20, 1e-21, 1e-22, 5e-23])
def test_subnormal_norm_narrows_or_widens_the_cone(scale):
    """|(u, v)| between ~2^-75 and ~1e-19: u*u + v*v is subnormal, so n1 = sqrt of it carries a relative error of up to
    tens of per cent and the reference's cone is cos > 0.9 * n1 / |(u, v)|, not cos > 0.9.  The predicate stays monotone
    along every row (no irregular pair), so the device plane must equal the oracle's outright; and the plane differs from
    the one of the same directions at unit scale once the norm error matters."""
    sc, sc1 = _tiny_dir_scene(scale, False), _tiny_dir_scene(1.0, False)
    ys, xs = np.nonzero(sc["label"][0] == 2)
    u, v = sc["vertex"][0, ys, xs, 6], sc["vertex"][0, ys, xs, 7]
    s2 = u * u + v * v
    assert (s2 < np.finfo(np.float32).tiny).all() and (s2 > 0).mean() > 0.5    # at 5e-23 some underflow to 0 outright
    rel = (np.sqrt(s2) / np.hypot(u.astype(np.float64), v.astype(np.float64)) - 1)[s2 > 0]
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], None, 0, -1.0, 0.02, 1, slack=True)
    _, dbg1 = oracle.hough_voting_gpu(sc1["label"], sc1["vertex"], sc1["extents"], sc1["meta"], None, 0, -1.0, 0.02, 1, debug=True)
    ndiff = int((dbg["votes"][0, 2] != dbg1["votes"][0, 2]).sum())
    print(f"scale {scale:g}: n1 relative error up to {np.abs(rel).max():.2e}; {ndiff} cells differ from unit scale; "
          f"{int(dbg['pairs'][0, 2, 1])} irregular of {int(dbg['pairs'][0, 2, 0])} pairs")
    assert dbg["pairs"][0, 2, 1] == 0 and dbg["pairs"][0, 2, 0] > 1000
    assert dbg["votes"][0, 2].max() > 50
    if scale <= 1e-21:
        assert np.abs(rel).max() > 1e-4 and ndiff > 0
