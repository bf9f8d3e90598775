"""Houghvotinggpu against the CPU oracle under the exactness criterion of DESIGN.md §3.3, at the benchmark's shapes, at every
k_vote band height and on planted edges of the vote predicate.

Planes: the device plane equals the oracle's (the reference's per-cell evaluation) wherever no irregular (sample, row) pair
reaches a cell, and differs by at most the number of such pairs elsewhere (tests/hough_ref.check_planes).  Rows: the op's
five outputs equal the oracle's (tests/util.assert_hough_rows_equal).  The band height and the end-point tolerance are the
library's defaults: the tests skip when PCNN_HOUGH_BAND_ROWS or PCNN_HOUGH_TAU0 overrides them, unless
PCNN_HOUGH_TEST_OVERRIDES=1 (`PCNN_HOUGH_TAU0=-1 PCNN_HOUGH_TEST_OVERRIDES=1` must fail the plane tests)."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from posecnn_b200 import synth
from tests import hough_ref as HR
from tests.util import assert_hough_rows_equal, to_np

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _library_defaults():
    """The asserted band heights and the criterion hold for the op's defaults.  PCNN_HOUGH_TEST_OVERRIDES=1 runs the tests
    under the overrides anyway, e.g. PCNN_HOUGH_TAU0=-1 (no end point re-checked), which must make the plane tests fail."""
    if os.environ.get("PCNN_HOUGH_TEST_OVERRIDES") == "1":
        return
    for k in ("PCNN_HOUGH_BAND_ROWS", "PCNN_HOUGH_TAU0", "PCNN_HOUGH_BAND_MIN"):
        if os.environ.get(k):
            pytest.skip(f"{k} overrides the op's defaults (PCNN_HOUGH_TEST_OVERRIDES=1 runs the test anyway)")


def _op():
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as op
    return op


def _dev(sc, dev):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    gt = t(sc["gt"]) if sc.get("gt") is not None and len(sc["gt"]) else None
    return t(sc["label"]), t(sc["vertex"]), t(sc["extents"]), t(sc["meta"]), gt


def _rows_and_status(sc, dev, is_train=0, skip=10, want=None):
    """The op's rows equal the oracle's; the status word is [0, 0] (no candidate overflow, every selected cell's scan vote
    equals its per-cell recount).  Returns the number of rows."""
    op = _op()
    lab, vert, ext, meta, gt = _dev(sc, dev)
    if want is None:
        want = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], sc.get("gt"), is_train, -1.0, 0.02,
                                       skip)
    got = op.hough_voting_gpu(lab, vert, ext, meta, gt, is_train, -1.0, 0.02, skip)
    assert_hough_rows_equal(got, want, is_train)
    status = op.hough_voting_gpu_capacity(lab, vert, ext, meta, gt, is_train, -1.0, 0.02, skip)[6]
    assert to_np(status)[:2].tolist() == [0, 0]
    return got[0].shape[0]


def _planes(sc, dev, skip=10, what=""):
    """Vote planes under the criterion; returns the summary dict."""
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], None, 0, -1.0, 0.02, skip, slack=True)
    lab, vert, ext, meta, _ = _dev(sc, dev)
    got = to_np(_op().hough_vote_planes(lab, vert, ext, meta, skip))
    return HR.check_planes(got, dbg, what)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the benchmark's frames at batch 32
# ---------------------------------------------------------------------------------------------------------------------
def test_bench_frames_batch32(cuda):
    """The 8 scenes of the `hough` workload tiled to batch 32 (16-row bands): every image's planes under the criterion
    against its scene's oracle planes, tiled copies bit-identical, and the batch's rows (cap 128 / 32 = 4 per image)."""
    op = _op()
    sc = HR.bench_scenes()
    B, (H, W), C = 32, sc["label"].shape[1:], 22
    R = HR.band_rows(B, H, W, C)
    assert R == 16
    sc32 = HR.tile(sc, B)
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], None, 0, -1.0, 0.02, 10, slack=True)
    lab, vert, ext, meta, _ = _dev(sc32, cuda)
    planes = op.hough_vote_planes(lab, vert, ext, meta, 10)
    n = HR.BENCH_FRAMES
    s = HR.check_planes(to_np(planes[:n]), dbg, "batch 32, images 0-7")
    for k in range(1, B // n):
        assert torch.equal(planes[k * n:(k + 1) * n], planes[:n]), f"images {k * n}-{(k + 1) * n - 1} differ from 0-{n - 1}"
    del planes
    rows = _rows_and_status(dict(sc32, gt=None), cuda)
    print(f"batch {B} x {H}x{W} x {C}: R = {R}; {s['pairs']} (sample, row) pairs, {s['irregular']} irregular, "
          f"{s['cells_differ']} cells differ (slack cells {s['slack_cells']}); {rows} rows")
    assert rows == 4 * B


# ---------------------------------------------------------------------------------------------------------------------
# 2. every band height
# ---------------------------------------------------------------------------------------------------------------------
def _wide_scene(B, H, W, C, seed):
    """Short, wide scene: an object near the left border, one in the middle and one whose window spans the whole width."""
    sc = HR.blank_scene(B, H, W, C, seed=seed)
    for b in range(B):
        HR.plant(sc, b, 1, 0.5 * W + 7 * b, H / 2, 45, H / 2 - 4, 1.0)
        HR.plant(sc, b, 2, 30, H / 2 + 2, 40, H / 2 - 5, 0.4)
        HR.plant(sc, b, 3, W - 60, H / 2 - 1, 50, H / 2 - 3, 0.15)     # window half-size ~1.6 x the image width
    return sc


BAND_CASES = {
    16: lambda: synth.make_scene(batch=24, height=256, width=256, num_classes=22, seed=77, other_channel_noise=False),
    8: lambda: _wide_scene(2, 96, 760, 6, 8),
    4: lambda: _wide_scene(1, 48, 1600, 4, 4),
    2: lambda: _wide_scene(1, 48, 3200, 4, 2),
    1: lambda: _wide_scene(1, 40, 6400, 4, 1),
}


@pytest.mark.parametrize("R", sorted(BAND_CASES, reverse=True))
def test_every_band_height(cuda, R):
    sc = BAND_CASES[R]()
    B, H, W = sc["label"].shape
    C = sc["extents"].shape[0]
    assert HR.band_rows(B, H, W, C) == R
    s = _planes(sc, cuda, what=f"R = {R}")
    rows = _rows_and_status(sc, cuda)
    widest = oracle.project_box(sc["extents"], sc["meta"][0], 3, 0.15) if R < 16 else 0.0
    print(f"{B} x {H}x{W} x {C}: R = {R}; {s['pairs']} pairs, {s['irregular']} irregular, {s['cells_differ']} cells differ; "
          f"{rows} rows; widest window half-size {widest:.0f}")
    assert s["max_vote"] > 10
    if R < 16:
        assert widest > W, "no class's window spans the image width"


# ---------------------------------------------------------------------------------------------------------------------
# 3. training rows at the training workload's shape
# ---------------------------------------------------------------------------------------------------------------------
def test_train_rows_batch64(cuda):
    """Batch 64 of the benchmark scenes with their gt poses, is_train = 1: 64 images x 2 ROIs x 9 jittered rows fill the
    1152-row capacity exactly; every row (boxes, poses, targets, weights, domain) equals the oracle's."""
    sc = HR.tile(HR.bench_scenes(), 64)
    B, H, W = sc["label"].shape
    R = HR.band_rows(B, H, W, 22)
    rows = _rows_and_status(sc, cuda, is_train=1)
    print(f"batch {B}, is_train = 1: R = {R}; {rows} rows, {len(sc['gt'])} gt poses")
    assert rows == 1152


# ---------------------------------------------------------------------------------------------------------------------
# 4. the low-resolution vertex source at batch 32
# ---------------------------------------------------------------------------------------------------------------------
def _lowres_from_scenes(sc, B, C, seed=11):
    """[B, H/8, W/8, 4C] head tensor whose vertex channels (C + 3c ..) hold dyadic directions from each 1/8-resolution cell
    to the planted object centre of class c and its log depth (random dyadic values for absent classes), plus a dyadic
    bias: pcnn_up8_heads' x8 bilinear up-sampling of it is exact in fp32."""
    rng = np.random.default_rng(seed)
    n, H, W = sc["label"].shape
    h, w = H // 8, W // 8
    low = (rng.integers(-64, 65, (B, h, w, 4 * C)) / 64.0).astype(np.float32)
    gy, gx = np.mgrid[0:h, 0:w] * 8.0 + 3.5
    for (b0, cls, cx, cy, z) in sc["centers"]:
        dx, dy = cx - gx, cy - gy
        nrm = np.sqrt(dx * dx + dy * dy) + 1e-6
        for b in range(b0, B, n):
            low[b, :, :, C + 3 * cls] = np.round(dx / nrm * 64) / 64
            low[b, :, :, C + 3 * cls + 1] = np.round(dy / nrm * 64) / 64
            low[b, :, :, C + 3 * cls + 2] = np.round(np.log(z) * 64) / 64
    bias = (rng.integers(-8, 9, 3 * C) / 128.0).astype(np.float32)
    bias[2::3] = 0
    return low, bias


def test_lowres_source_batch32(cuda):
    from posecnn_b200 import heads
    op = _op()
    sc = HR.bench_scenes()
    B, C = 32, 22
    sc32 = HR.tile(sc, B)
    H, W = sc32["label"].shape[1:]
    low_np, bias_np = _lowres_from_scenes(sc, B, C)
    lowres, bias = torch.from_numpy(low_np).to(cuda), torch.from_numpy(bias_np).to(cuda)
    lab = torch.from_numpy(sc32["label"]).to(cuda)
    ext = torch.from_numpy(sc32["extents"]).to(cuda)
    meta = torch.from_numpy(np.ascontiguousarray(sc32["meta"])).to(cuda)
    zero_bias = torch.zeros(C, device=cuda)
    dense = heads.up8_heads(lowres, zero_bias, bias, vertex=True)[1]
    full = op.hough_voting_gpu_capacity(lab, dense, ext, meta, None, 0, -1.0, 0.02, 10)
    low = op.hough_voting_gpu_capacity(lab, None, ext, meta, None, 0, -1.0, 0.02, 10, lowres=lowres, bias_vertex=bias)
    names = ("box", "pose", "target", "weight", "domain", "num_rois", "status")
    for name, a, b in zip(names, full, low):
        assert torch.equal(a, b), f"lowres source: {name} differs from the dense source"
    assert to_np(full[6])[:2].tolist() == [0, 0]
    nr = int(full[5].item())
    box = to_np(full[0])
    for off, n in ((0, 16), (16, 16), (0, 8), (8, 24)):
        shard = op.hough_voting_gpu_capacity(lab[off:off + n], None, ext, meta[off:off + n], None, 0, -1.0, 0.02, 10,
                                             lowres=lowres[off:off + n], bias_vertex=bias, batch_global=B, batch_offset=off)
        sel = np.nonzero((box[:nr, 0] >= off) & (box[:nr, 0] < off + n))[0]
        lo, hi = (int(sel[0]), int(sel[-1]) + 1) if sel.size else (0, 0)
        assert hi - lo == sel.size
        assert int(shard[5].item()) == hi - lo, (off, n)
        for name, a, b in zip(names[:5], full[:5], shard[:5]):
            assert torch.equal(a[lo:hi], b[:hi - lo]), f"shard [{off}, {off + n}): {name}"
            assert not b[hi - lo:].any(), f"shard [{off}, {off + n}): {name} beyond its rows"
        assert to_np(shard[6])[:2].tolist() == [0, 0]
    dense_sc = dict(sc32, vertex=to_np(dense), gt=None)
    del dense
    rows = _rows_and_status(dense_sc, cuda)
    print(f"lowres source, batch {B}: R = {HR.band_rows(B, H, W, C)}; {nr} rows, bit-identical to the dense source, "
          f"whole batch and 4 shardings")
    assert rows == nr == 4 * B


# ---------------------------------------------------------------------------------------------------------------------
# 5. planted edges of the predicate
# ---------------------------------------------------------------------------------------------------------------------
def _edge_scene(case):
    H, W, C = 64, 96, 4
    sc = HR.blank_scene(1, H, W, C, seed=sum(map(ord, case)))
    ys, xs = HR.plant(sc, 0, 1, 30, 30, 18, 14, 0.8)                     # a regular object in every scene
    v = sc["vertex"][0]
    regular = True                                                       # the scene is built to have no irregular pair
    if case == "underflow":
        ys, xs = HR.plant(sc, 0, 2, 70, 34, 16, 16, 0.7)
        v[ys, xs, 6:8] *= np.float32(1e-24)                              # u*u + v*v underflows: n1 = 0, dot != 0
        v[ys[::7], xs[::7], 6] = 0.0                                     # u = 0: whole rows on v's side
        v[ys[3::14], xs[3::14], 7] = 0.0                                 # v = 0
        v[ys[5::9], xs[5::9], 6:8] *= np.float32(2.0 ** -60)            # subnormal components
    elif case.startswith("subnormal"):
        ys, xs = HR.plant(sc, 0, 2, 70, 34, 16, 16, 0.7)
        v[ys, xs, 6:8] *= np.float32(case.split("-", 1)[1])              # u*u + v*v subnormal: n1 off by up to ~30%
        v[ys[::7], xs[::7], 6] = 0.0
    elif case == "zero":
        ys, xs = HR.plant(sc, 0, 2, 70, 34, 16, 16, 0.7)
        v[ys[::3], xs[::3], 6:8] = 0.0                                   # exactly zero directions: no votes
        v[ys[1::3], xs[1::3], 6] = -0.0
        v[ys[1::3], xs[1::3], 7] = 0.0
    elif case == "near_threshold":
        regular = False
        ys, xs = HR.plant(sc, 0, 2, 66, 36, 20, 16, 0.5)
        d = HR.near_threshold_dirs(count=8)
        k = np.arange(d.shape[0]) * (xs.size // d.shape[0])
        v[ys[k], xs[k], 6], v[ys[k], xs[k], 7] = d[:, 0], d[:, 1]
    elif case == "axes":
        regular = False                                                  # the half-angle directions sit on the threshold
        ys, xs = HR.plant(sc, 0, 2, 66, 36, 20, 16, 0.6)
        ca, sa = np.float32(0.9), np.sqrt(np.float32(1) - np.float32(0.9) * np.float32(0.9))
        dirs = [(1, 0), (-1, 0), (0, 1), (0, -1), (ca, sa), (ca, -sa), (-ca, sa), (-ca, -sa), (sa, ca), (-sa, ca), (sa, -ca),
                (-sa, -ca)]
        for i, (a, b) in enumerate(dirs):
            for j, scale in enumerate((1.0, 3.7, 1e-3, 1e-18)):
                p = 1 + 4 * (4 * i + j)
                v[ys[p], xs[p], 6], v[ys[p], xs[p], 7] = np.float32(a) * np.float32(scale), np.float32(b) * np.float32(scale)
    elif case == "borders":
        for cls, (cx, cy) in zip((1, 2, 3), ((8, 6), (W - 6, 8), (W - 9, H - 6))):
            sc["label"][0][sc["label"][0] == cls] = 0
            HR.plant(sc, 0, cls, cx, cy, 22, 18, 0.35)                   # windows clipped by the image borders
        HR.plant(sc, 0, 1, 10, H - 8, 16, 14, 0.3)
        HR.plant(sc, 0, 3, 48, 32, 12, 14, 0.12)                          # window wider than the image
        assert oracle.project_box(sc["extents"], sc["meta"][0], 3, 0.12) > W
    elif case == "depth":
        ys, xs = HR.plant(sc, 0, 2, 66, 36, 20, 16, 0.6)
        sc["extents"][2] = (0.1, 0.12, 2.0)                              # half extent 1 = exp(0): Z = d - 1 is exactly 0
        zs = np.float32([0.0, -0.5, -3.0, -np.inf, 0.3])                 # d = 1, 0.61, 0.05, 0 and one regular depth
        v[ys[::2], xs[::2], 8] = np.resize(zs, ys[::2].size)            # project_box divides by Z = 0 or Z < 0
    return sc, regular


EDGE_CASES = ("underflow", "subnormal-1e-20", "subnormal-1e-21", "subnormal-1e-22", "subnormal-5e-23", "zero", "near_threshold", "axes",
              "borders", "depth")


@pytest.mark.parametrize("case", EDGE_CASES)
def test_predicate_edges(cuda, case):
    sc, regular = _edge_scene(case)
    _, dbg = oracle.hough_voting_gpu(sc["label"], sc["vertex"], sc["extents"], sc["meta"], None, 0, -1.0, 0.02, 1, slack=True)
    irregular = int(dbg["pairs"][..., 1].sum())
    if regular:
        assert irregular == 0, f"{case}: the scene was built without irregular pairs"
    lab, vert, ext, meta, _ = _dev(sc, cuda)
    got = to_np(_op().hough_vote_planes(lab, vert, ext, meta, 1))
    s = HR.check_planes(got, dbg, case)
    if regular:
        np.testing.assert_array_equal(got, dbg["votes"])
    if case == "underflow" or case.startswith("subnormal"):
        assert dbg["votes"][0, 2].max() > 50                              # the tiny directions vote in the reference
    if case in ("near_threshold", "axes"):
        assert irregular > 0
    B, H, W = sc["label"].shape
    rows = _rows_and_status(sc, cuda, skip=1)
    print(f"{case}: R = {HR.band_rows(B, H, W, sc['extents'].shape[0])}; {s['pairs']} pairs, {irregular} irregular, "
          f"{s['cells_differ']} cells differ; {rows} rows")
    assert rows >= 2
