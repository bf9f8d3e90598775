"""The references of tests/vertex_loss_ref.py checked without a GPU: against independent float32 / float64 computations in
another order, against the oracle's restatements of the data layer and of smooth_l1_loss_vertex, and the exactness checks
(log-z midpoints, exact square sums, the loss's straddle check) firing on crafted inputs."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import oracle
from tests import vertex_loss_ref as V
from tests.train_coord_ref import vertex_targets_3d


def _problem(coord, C=6, sigma=1.0, B=2, H=128, W=192, seed=0, w_inside=1.0):
    return V.loss_problem(B, H, W, C, coord, sigma, torch.Generator().manual_seed(seed), w_inside=w_inside)


def test_logz_table_and_midpoint_check():
    """LOGZ_TABLE passes; the check fires on a crafted threshold, and the helper flags an exact fp32 midpoint."""
    lz = V.check_log_midpoints(V.LOGZ_TABLE)
    assert np.array_equal(lz, np.log(V.LOGZ_TABLE.astype(np.float64)).astype(np.float32))
    assert V.near_f32_midpoint(np.array([1.0 + 2.0 ** -24, 3.0 + 2.0 ** -23]))[0]                 # exact midpoints
    assert V.near_f32_midpoint(np.nextafter(1.0 + 2.0 ** -24, 2.0)) and V.near_f32_midpoint(3.0 + 2.0 ** -23)
    assert not V.near_f32_midpoint(np.array([1.0, 1.0 + 2.0 ** -23])).any()
    with pytest.raises(V.MidpointTooClose):
        V.check_log_midpoints(np.float32([0.75]), ulps=2 ** 26)          # log 0.75 lies ~2^24 double ulps from a midpoint


def test_square_sum_check_fires():
    V.check_square_sums_exact(np.float32([-63.5, 700.25]), np.float32([0.0, 511.75]), 480, 640)
    with pytest.raises(AssertionError, match="2\\^-12"):
        V.check_square_sums_exact(np.float32([1e-5]), np.float32([0.0]), 480, 640)
    with pytest.raises(AssertionError, match="2\\^11"):
        V.check_square_sums_exact(np.float32([3000.0]), np.float32([0.0]), 480, 640)


def test_exact_sum():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(10000).astype(np.float32) * np.float32(1e6),
                        rng.standard_normal(10000).astype(np.float32) * np.float32(1e-30), np.float32([2.0 ** -149, 0.0])])
    assert V.exact_sum(x) == sum((Fraction(float(v)) for v in x), Fraction(0))
    assert float(V.exact_sum(x)) == math.fsum(x.astype(np.float64).tolist())


@pytest.mark.parametrize("C", [6, 2])
def test_targets_2d_against_oracle_and_torch(C):
    """targets_2d == oracle.generate_vertex_targets (direction channels bit for bit, log z equal: the table's logs are the
    same numpy call), and the direction channels equal a torch float64 computation with hypot, bit for bit."""
    P = _problem(False, C)
    listed, cls, t = V.targets_2d(P["label"], P["centers"])
    tg, wt = V.dense(listed, cls, t, C, 10.0)
    otg, owt = oracle.generate_vertex_targets(P["label"], P["centers"], 10.0)
    assert np.array_equal(wt, owt) and np.array_equal(tg, otg)
    B, H, W = listed.shape
    cen = torch.as_tensor(P["centers"]).double()[torch.arange(B)[:, None, None], torch.as_tensor(cls)]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    dx, dy = cen[..., 0] - xs, cen[..., 1] - ys
    nrm = torch.hypot(dy, dx) + 1e-10                                  # correctly rounded: equals sqrt of the exact sum
    lst = torch.as_tensor(listed)
    assert torch.equal((dx / nrm).float()[lst], torch.as_tensor(t[..., 0])[lst])
    assert torch.equal((dy / nrm).float()[lst], torch.as_tensor(t[..., 1])[lst])


def test_targets_3d_against_golden_restatement_and_torch():
    """targets_3d == train_coord_ref.vertex_targets_3d (the reference's float32 _scale_vertmap) and a torch float32
    computation of (v - vmin) / span as a v + b, bit for bit."""
    C = 6
    P = _problem(True, C)
    listed, cls, t = V.targets_3d(P["label"], P["vertmap"], P["centers"], P["extents"])
    tg, wt = V.dense(listed, cls, t, C, 10.0)
    gt, gw = vertex_targets_3d(P["label"], P["vertmap"], P["centers"], P["extents"], 10.0)
    assert np.array_equal(wt, gw) and np.array_equal(tg, gt)
    e = torch.as_tensor(P["extents"])
    span = e / 2 - (-e / 2)
    a = torch.where(span > 0, 1 / span.clamp(min=1e-30), torch.zeros(()))
    b = torch.where(span > 0, (e / 2) / span.clamp(min=1e-30), torch.zeros(()))
    c = torch.as_tensor(cls)
    want = torch.as_tensor(P["vertmap"]) * a[c] + b[c]
    lst = torch.as_tensor(listed)
    assert torch.equal(want[lst], torch.as_tensor(t)[lst])


def test_targets_3d_operands_round():
    """On the generated 3-D operands the float32 operations of coord_scale / coord_target round: a target formed with one
    fused multiply-add (fmaf(a, v, b)) or as (v - vmin) / span differs from the op-by-op restatement on many listed values,
    so a kernel that fused or reordered them would fail the bit-exact target and loss tests."""
    from tests.pose_bwd_ref import fmaf
    C = 22
    P = _problem(True, C, B=1, H=480, W=640)
    listed, cls, t = V.targets_3d(P["label"], P["vertmap"], P["centers"], P["extents"])
    ab = V.R.coord_scale(torch.as_tensor(P["extents"]))[torch.as_tensor(cls)]
    v = torch.as_tensor(P["vertmap"])
    fused = fmaf(ab[..., 0], v, ab[..., 1]).numpy()
    e = torch.as_tensor(P["extents"])[torch.as_tensor(cls)]
    vmin = -e / 2
    span = e / 2 - vmin
    reordered = torch.where(span > 0, (v - vmin) / torch.where(span > 0, span, torch.ones(())), torch.zeros(())).numpy()
    n = int(listed.sum()) * 3
    n_fused = int((fused != t)[listed].sum())
    n_reordered = int((reordered != t)[listed].sum())
    print(f"{n} listed target values: fmaf(a, v, b) differs on {n_fused}, (v - vmin) / span on {n_reordered}")
    assert n_fused > n // 20 and n_reordered > n // 20


def test_targets_instances_against_oracle():
    """targets_instances == oracle.generate_vertex_targets_instances (in-order overwrite: the last matching instance
    wins; z <= 0 unused), with a repeated (class, mask id) and an unused slot that matches pixels."""
    rng = np.random.default_rng(3)
    B, H, W, C = 2, 40, 56, 5
    label = rng.integers(-1, C + 2, (B, H, W)).astype(np.int32)
    mask = rng.integers(0, 3, (B, H, W)).astype(np.int32)
    inst = np.zeros((B, 5, 5), np.float32)
    for i, (c, m) in enumerate([(1, 1), (2, 1), (1, 2), (1, 1), (3, 2)]):
        inst[:, i] = (c, m, rng.integers(0, W * 4096) / 4096, rng.integers(0, H * 4096) / 4096, V.LOGZ_TABLE[i])
    inst[:, 2, 4] = 0.0
    listed, cls, t = V.targets_instances(label, mask, inst, C)
    tg, wt = V.dense(listed, cls, t, C, 10.0)
    otg, owt = oracle.generate_vertex_targets_instances(label, mask, inst, C, 10.0)
    assert np.array_equal(wt, owt) and np.array_equal(tg, otg)
    assert not ((label == 1) & (mask == 2) & listed).any() and ((label == 1) & (mask == 1) & listed).any()


def test_sl1_terms_against_oracle_expression():
    """sl1_terms == the oracle's float32 masked-sum form of the same smooth L1, bit for bit, with boundary values."""
    rng = np.random.default_rng(1)
    for sigma in (1.0, 2.5):
        s2 = np.float32(sigma) ** 2
        p = rng.standard_normal(20000).astype(np.float32)
        t = rng.standard_normal(20000).astype(np.float32)
        t[:100] = 0
        p[:50], p[50:100] = np.float32(1) / s2, -(np.float32(1) / s2)
        got = V.sl1_terms(p, t, 1.0, sigma)
        diff = p - t
        ad = np.abs(diff)
        sign = (ad < np.float32(1.0) / s2).astype(np.float32)
        want = diff * diff * (s2 / np.float32(2)) * sign + (ad - np.float32(0.5) / s2) * (np.float32(1) - sign)
        assert np.array_equal(got, want)
        # at |diff| == 1 / sigma^2 the two branches agree in fp32 at these sigmas (the forward loss cannot see the branch)
        d = np.float32(1) / s2
        assert d * d * (s2 * np.float32(0.5)) == d - np.float32(0.5) / s2


@pytest.mark.parametrize("coord", [False, True], ids=["2d", "3d"])
@pytest.mark.parametrize("sigma", [1.0, 2.5])
def test_loss_reference_against_oracle_and_float64(coord, sigma):
    """The expected output equals float32 of a float64 torch sum in sorted order (no straddle here), and agrees with
    oracle.smooth_l1_loss_vertex on the dense blobs and the dense float64 prediction within 1e-6 relative."""
    C = 6
    P = _problem(coord, C, sigma, seed=int(4 * sigma) + coord)
    ref = V.reference(P)
    assert ref["boundary"] > 0 and ref["count"] > 0
    terms = torch.as_tensor(ref["terms"]).double().sort().values
    assert np.float32(float(terms.sum()) / (float(ref["out1"]) + 1e-10)) == ref["out0"]
    assert ref["out1"] == np.float32(3 * ref["count"] * P["w_inside"])
    tg, wt = V.dense(ref["listed"], ref["cls"], ref["t"], C, P["w_inside"])
    pv = (V.R.up(P["lowres"][..., C:], 8) + P["bias_v"].double()).float().numpy()
    want, _ = oracle.smooth_l1_loss_vertex(pv, tg, wt, sigma)
    assert abs(float(ref["out0"]) - want) <= 1e-6 * abs(want)


def test_straddle_check_fires():
    """A term sum whose quotient by the weight sum is an fp32 midpoint raises Straddle; a value off the midpoint does not.
    One listed pixel, w_inside = 2^20 (so the 1e-10 vanishes from the weight sum 3 2^20), sigma 1, predictions 0: targets
    -3 and -1.1875 2^-20 give linear terms 3 2^20 - 1/2 and 0.6875, whose sum over 3 2^20 is 1 + 2^-24."""
    w = 2.0 ** 20
    listed = np.ones((1, 1, 1), bool)
    pred = np.zeros((1, 1, 1, 3), np.float32)
    targ = np.float32([-3.0, -1.1875 * 2.0 ** -20, 0.0]).reshape(1, 1, 1, 3)
    assert V.sl1_terms(pred[listed], targ[listed], w, 1.0).tolist() == [[3 * w - 0.5, 0.6875, 0.0]]
    with pytest.raises(V.Straddle):
        V.loss_vertex(pred, targ, listed, w, 1.0)
    targ[..., 1] = 0
    L = V.loss_vertex(pred, targ, listed, w, 1.0)
    assert L["out0"] == np.float32((3 * w - 0.5) / (3 * w)) and L["out1"] == np.float32(3 * w)


def test_budget_check_fires():
    P = _problem(False, 6)
    listed, cls, _ = V.targets_2d(P["label"], P["centers"])
    big = P["lowres"].clone()
    big[..., 6:] *= 2 ** 8
    with pytest.raises(V.BudgetExceeded):
        V.own_vertex_values(big, P["bias_v"], cls, 6, P["unit"])


def test_pack_pose_meta_reference_against_oracle():
    """pack_pose_meta == oracle.pack_pose_meta: image, class, box and translation columns bit for bit, quaternions (scipy vs
    the oracle's eigenvector) within 2e-7, meta within 2^-23 relative (the cofactor inverse vs pinv; pinv leaves ~1e-19 where
    the inverse is exactly 0)."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(2)
    B, I = 3, 6
    cls = np.where(rng.random((B, I)) < 0.3, -1, rng.integers(1, 22, (B, I))).astype(np.int32)
    poses = np.zeros((B, I, 3, 4), np.float32)
    poses[..., :3] = Rotation.random(B * I, random_state=1).as_matrix().reshape(B, I, 3, 3)
    poses[..., 3] = rng.uniform(-1, 1, (B, I, 3))
    K = np.zeros((B, 3, 3), np.float32)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 1066.75, 1067.5, 312.9921875, 241.3125, 1
    for scale, flip in ((1.0, False), (0.5, True)):
        blob, n, meta = V.pack_pose_meta(poses, cls, K, scale, flip)
        ob, om = oracle.pack_pose_meta(poses, cls, K, scale, flip)
        assert n == ob.shape[0] and not blob[n:].any()
        assert np.array_equal(blob[:n, :6], ob[:, :6]) and np.array_equal(blob[:n, 10:], ob[:, 10:])
        np.testing.assert_allclose(blob[:n, 6:10], ob[:, 6:10], rtol=0, atol=2e-7)
        np.testing.assert_allclose(meta, om, rtol=2 ** -23, atol=1e-9)            # pinv leaves ~1e-19 where 0 is exact
