"""Colour-only object-coordinate pose estimation on the GPU (csrc/coord_pose.cu k_sample2d / k_ransac<true>, DESIGN.md §13)
against the float64 restatement tests/coord_pose2d_ref.py on analytic 480x640 scenes: hypotheses (class, attempts, four pixels)
and per-round subsets exactly, counts and survivors, final poses; dense and low-resolution sources bit-identical; shards,
determinism, CUDA-graph replay; the depth estimator's subsets on hole-free images; edge cases; the synthesizer-style wrapper; the
network's estimate_rgb outputs and the refinement of its depth estimate.  Measured deltas are printed (DESIGN.md §13 records
them)."""
import numpy as np
import pytest
import torch

from posecnn_b200 import synth
from posecnn_b200.coord_pose import CoordPoseEstimator, assemble_records, estimate_poses_2d, estimate_poses_3d
from tests import coord_pose2d_ref as ref2
from tests import coord_pose_ref as ref
from tests.test_coord_pose_cpu import rot_err_deg

pytestmark = pytest.mark.gpu
KEYS = [0x1234567890ABCDEF, 77, 2**63 + 5, 31337]


def scene(B, C, seed, noise=0.0, outliers=0.0):
    return synth.make_coordinate_scene(batch=B, num_classes=C, objects_per_image=3 if C > 2 else 1, seed=seed, coord_noise_m=noise,
                                       outlier_fraction=outliers)


def keys_of(keys, B, cuda):
    return torch.tensor(np.array(keys[:B], np.uint64).view(np.int64), device=cuda)


def run(sc, cuda, keys, trace=False, **kw):
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    B = sc["label"].shape[0]
    src = kw.pop("src", None) or dict(vertex=T(sc["vertex"]))
    return estimate_poses_2d(T(sc["label"]), T(sc["meta"]), T(sc["extents"]), keys_of(keys, B, cuda), trace=trace, **src, **kw)


def rot_diff_deg(Ra, Rb):
    """Angle between two rotations from |Ra - Rb|_F = 2 sqrt(2) sin(angle / 2): unlike the arccos of the trace, it resolves the
    1e-7 rounding of a float32 matrix (the arccos form bottoms out near 0.01 deg there)."""
    return float(np.degrees(2.0 * np.arcsin(min(1.0, np.linalg.norm(Ra - Rb) / (2.0 * np.sqrt(2.0))))))


def host(out):
    return {k: v.cpu().numpy() for k, v in out.items()}


def cam_of(sc, b):
    return (sc["meta"][b, 0], sc["meta"][b, 4], sc["meta"][b, 2], sc["meta"][b, 5])


@pytest.mark.parametrize("B,C,noise,outliers,seed", [(1, 22, 0.0, 0.0, 3), (2, 22, 0.002, 0.2, 4), (1, 2, 0.0, 0.2, 5),
                                                     (4, 2, 0.002, 0.0, 6)])
def test_against_oracle(cuda, B, C, noise, outliers, seed):
    sc = scene(B, C, seed, noise, outliers)
    out = host(run(sc, cuda, KEYS, trace=True))
    worst = dict(rot=0.0, trans=0.0, count=0, objects=0)
    for b in range(B):
        want = ref2.estimate_image(sc["label"][b], sc["vertex"][b], sc["extents"], cam_of(sc, b), KEYS[b], C)
        th = out["trace_hyp"][b]
        for h, hy in enumerate(want["hyps"]):          # drawn objects, attempts and four-pixel draws: exact
            assert (th[h, 0], th[h, 1]) == (hy["obj"], hy["attempts"]), (b, h)
            assert list(th[h, 2:6]) == (hy["pix"] if hy["obj"] else [-1] * 4), (b, h)
        np.testing.assert_array_equal(out["info"][b][:, [0, 1, 3, 4]], want["info"][:, [0, 1, 3, 4]])
        for c, rounds in want["rounds"].items():
            worst["objects"] += 1
            tr = out["trace_round"][b, c]
            for r, rd in enumerate(rounds):              # subsets: exact; counts within the pairs at the gate
                assert tr[r, 0] == rd["taken"] and (int(tr[r, 1]) & 0xFFFFFFFF) == rd["hash"], (b, c, r)
                assert tr[r, 2] == rd["best"], (b, c, r)
                worst["count"] = max(worst["count"], abs(int(tr[r, 3]) - rd["best_count"]))
                assert abs(int(tr[r, 3]) - rd["best_count"]) <= rd["near"][rd["best"]], (b, c, r)
            assert out["info"][b, c, 5] == want["info"][c, 5], (b, c)        # survivor
            worst["rot"] = max(worst["rot"], rot_diff_deg(out["poses"][b, c, :, :3].astype(np.float64), want["poses"][c, :, :3]))
            worst["trans"] = max(worst["trans"], float(np.linalg.norm(out["poses"][b, c, :, 3] - want["poses"][c, :, 3])))
        for c in range(C):
            if c not in want["rounds"]:
                assert not out["poses"][b, c].any()
    print(f"\n[coord_pose2d oracle] B={B} C={C} noise={noise} outliers={outliers}: {worst}")
    # float32 output of a float64 pose: ~1e-7 relative
    assert worst["rot"] < 1e-3 and worst["trans"] < 1e-5 and worst["objects"] >= 1


def test_planted_recovery(cuda):
    sc = scene(2, 22, 11)
    out = host(run(sc, cuda, KEYS))
    worst_r = worst_t = 0.0
    n = 0
    for row in sc["poses"]:
        b, c = int(row[0]), int(row[1])
        if (sc["label"][b] == c).sum() <= ref.MIN_AREA:
            assert not out["poses"][b, c].any()
            continue
        worst_r = max(worst_r, rot_err_deg(out["poses"][b, c, :, :3].astype(np.float64), synth.quat_to_rot(row[2:6])))
        worst_t = max(worst_t, float(np.linalg.norm(out["poses"][b, c, :, 3] - row[6:9])))
        n += 1
    print(f"\n[coord_pose2d planted] {n} objects: worst {worst_r:.4f} deg, {1000 * worst_t:.3f} mm")
    assert n >= 3 and worst_r < 0.5 and worst_t < 0.002


def test_per_hypothesis_counts_against_oracle(cuda):
    """Every hypothesis's inlier count in every round, within the number of its pairs whose distance lies within 1e-6 relative
    of the 10 px gate."""
    sc = scene(1, 22, 29, 0.002, 0.2)
    out = host(run(sc, cuda, KEYS, trace=True))
    want = ref2.estimate_image(sc["label"][0], sc["vertex"][0], sc["extents"], cam_of(sc, 0), KEYS[0], 22)
    th = out["trace_hyp"][0]
    compared = 0
    for c, rounds in want["rounds"].items():
        for r, rd in enumerate(rounds):
            for h, n in rd["counts"].items():
                assert abs(int(th[h, 6 + r]) - n) <= rd["near"][h], (c, r, h)
                compared += 1
    counted = {(h, r) for rounds in want["rounds"].values() for r, rd in enumerate(rounds) for h in rd["counts"]}
    for h in range(ref.NUM_HYP):
        for r in range(ref.ROUNDS):
            if (h, r) not in counted:
                assert th[h, 6 + r] == -1
    assert compared >= 256


def test_lowres_source_bit_identical_to_dense(cuda):
    from posecnn_b200 import heads
    B, C = 2, 22
    sc = scene(B, C, 13)
    h, w = 60, 80
    lowres = np.zeros((B, h, w, 4 * C), np.float32)
    lowres[..., C:] = sc["vertex"][:, 4::8, 4::8]
    lr = torch.from_numpy(lowres).to(cuda)
    bv = torch.full((3 * C,), 0.01, device=cuda)
    bs = torch.zeros(C, device=cuda)
    dense = heads.up8_heads(lr, bs, bv, vertex=True, prob=True, score=True)[1]
    a = run(sc, cuda, KEYS, trace=True, src=dict(vertex=dense))
    b = run(sc, cuda, KEYS, trace=True, src=dict(lowres=lr, bias_vertex=bv))
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert (a["info"][..., 1] > 0).any()


def test_shard_determinism_and_graph(cuda):
    sc = scene(4, 22, 17, 0.002, 0.2)
    whole = run(sc, cuda, KEYS, trace=True)
    again = run(sc, cuda, KEYS, trace=True)
    for k in whole:
        assert torch.equal(whole[k], again[k]), k
    part = {k: sc[k][2:4] for k in ("label", "meta", "vertex")}
    part["extents"] = sc["extents"]
    shard = run(part, cuda, KEYS[2:], trace=True)
    for k in whole:
        assert torch.equal(whole[k][2:4], shard[k]), k
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    inp = dict(label=T(sc["label"]), meta=T(sc["meta"]), ext=T(sc["extents"]), vertex=T(sc["vertex"]), keys=keys_of(KEYS, 4, cuda))
    f = lambda: estimate_poses_2d(inp["label"], inp["meta"], inp["ext"], inp["keys"], vertex=inp["vertex"], trace=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = f()
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for k in whole:
            assert torch.equal(res[k], whole[k]), k


def test_hole_free_subsets_equal_the_depth_estimators(cuda):
    sc = scene(2, 22, 31, 0.002, 0.0)
    sc["depth"] = np.where(sc["depth"] == 0, 1.0, sc["depth"]).astype(np.float32)      # no hole anywhere
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rgb = host(run(sc, cuda, KEYS, trace=True))
    d3 = host(estimate_poses_3d(T(sc["label"]), T(sc["depth"]), T(sc["meta"]), T(sc["extents"]), keys_of(KEYS, 2, cuda),
                                vertex=T(sc["vertex"]), trace=True))
    both = (rgb["info"][..., 1] > 0) & (d3["info"][..., 1] > 0)
    assert both.sum() >= 3
    np.testing.assert_array_equal(rgb["trace_round"][both][..., :2], d3["trace_round"][both][..., :2])
    np.testing.assert_array_equal(rgb["info"][..., 0], d3["info"][..., 0])


def test_edge_cases_give_zero_rows(cuda):
    C = 6
    sc = scene(4, C, 19)
    small = int(sc["poses"][0, 1])
    keep = np.argwhere(sc["label"][0] == small)[:300]
    sc["label"][0][sc["label"][0] == small] = 0
    sc["label"][0][keep[:, 0], keep[:, 1]] = small                # <= 400 pixels
    zero_c = [int(r[1]) for r in sc["poses"] if r[0] == 0 and int(r[1]) != small and (sc["label"][0] == int(r[1])).sum() > 400]
    assert zero_c, "the scene must hold a second object for the zero-extents case"
    sc["extents"] = sc["extents"].copy()
    sc["extents"][zero_c[0]] = 0.0
    sc["vertex"] = sc["vertex"].copy()
    sc["vertex"][1] = 0.0                                         # image 1: every coordinate empty
    sc["label"][2] = 0                                            # image 2: no object
    out = host(run(sc, cuda, KEYS))
    assert not out["poses"][1].any() and (out["info"][1, 1:, 4] == 256).all()
    assert not out["poses"][2].any() and (out["info"][2, :, 1] == 0).all() and (out["info"][2, :, 4] == 0).all()
    assert not out["poses"][0, small].any() and out["info"][0, small, 0] <= 400
    assert not out["poses"][0, zero_c[0]].any() and out["info"][0, zero_c[0], 1] == 0
    for c in [c for c in range(1, C) if not (sc["label"][0] == c).any()]:
        assert not out["poses"][0, c].any() and out["info"][0, c, 5] == -1
    assert (out["info"][..., 3] == -1).all()
    assert out["poses"][3].any()                                  # the untouched image still gets poses


def test_wrapper_equals_batched_rows(cuda):
    C = 22
    sc = scene(1, C, 23, 0.002, 0.2)
    out = host(run(sc, cuda, KEYS))
    poses = np.zeros((3, 4, C), np.float32)
    m = sc["meta"][0]
    CoordPoseEstimator(key=KEYS[0]).estimate_poses_2d(sc["label"][0], sc["vertex"][0], sc["extents"], poses, C, m[0], m[4], m[2], m[5])
    np.testing.assert_array_equal(poses, out["poses"][0].transpose(1, 2, 0))
    assert poses[2, 3].any()


def test_network_estimate_rgb_eager_graph_refine_and_guards(cuda):
    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    from posecnn_b200.pose_refine import refine_poses
    C, B, H, W = 6, 2, 128, 160
    net = vgg16_convs(num_classes=C, device=cuda, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False,
                      scales=(1.5,)).init_random(seed=0, bias_std=0.05)
    rgb, depth_m = synth.make_images(B, H, W, seed=3)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    data, meta, ext = T(rgb), T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)), T(synth.extents_for(C))
    depth = T((depth_m * 10000.0).astype(np.float32))
    pts = T(synth.make_model_points(C, 256))
    keys = torch.tensor([3, 9], dtype=torch.int64, device=cuda)
    off = {k: v.clone() for k, v in net.forward(data, meta, ext, dense_vertex=False).items()}
    on = {k: v.clone() for k, v in net.forward(data, meta, ext, dense_vertex=False, estimate_keys=keys, estimate_rgb=True).items()}
    new = {"estimate_poses_rgb", "estimate_info_rgb", "detections_rois_rgb", "detections_poses_rgb", "num_detections_rgb"}
    assert set(on) - set(off) == new and set(off) <= set(on)
    for k in off:
        assert torch.equal(off[k], on[k]), k
    assert on["estimate_info_rgb"][..., 0].sum() > 0
    est = estimate_poses_2d(on["label_2d"], meta, ext, keys, lowres=net._last_lowres, bias_vertex=net.params["vertex_pred/biases"])
    assert torch.equal(est["poses"], on["estimate_poses_rgb"]) and torch.equal(est["info"], on["estimate_info_rgb"])
    rr, pp, nn = assemble_records(est["poses"], ext, meta, 1.5, 0)
    assert torch.equal(rr, on["detections_rois_rgb"]) and torch.equal(pp, on["detections_poses_rgb"])
    assert torch.equal(nn, on["num_detections_rgb"])
    # both estimates and the refinement of the depth estimate, eager
    kw = dict(dense_vertex=False, estimate_keys=keys, estimate_rgb=True, estimate_depth=depth, refine_depth=depth, refine_points=pts)
    full = {k: v.clone() for k, v in net.forward(data, meta, ext, **kw).items()}
    for k in new:
        assert torch.equal(full[k], on[k]), k
    refined = refine_poses(full["label_2d"], depth, meta, torch.nn.functional.pad(full["detections_rois"], (0, 1)),
                           full["detections_poses"], pts, num_rows=full["num_detections"])
    for k, v in (("detections_poses_refined", "poses_refined"), ("detections_poses_icp", "poses_icp"), ("detections_icp_info", "icp_info")):
        assert torch.equal(full[k], refined[v]), k
    # graphed
    gf = GraphedForward(net, data, meta, ext, **kw)
    L = gf(data, meta, refine_depth=depth, estimate_depth=depth)
    torch.cuda.synchronize()
    for k in new | {"estimate_poses", "detections_rois", "detections_poses_refined", "detections_poses_icp", "detections_icp_info"}:
        assert torch.equal(L[k], full[k]), k
    gf0 = GraphedForward(net, data, meta, ext, dense_vertex=False)
    L0 = gf0(data, meta)
    torch.cuda.synchronize()
    assert not (set(L0) & new)
    # guards
    net2d = vgg16_convs(num_classes=C, device=cuda).init_random(seed=0)
    with pytest.raises(ValueError, match="vertex_reg_3d"):
        net2d.forward(data, meta, ext, estimate_rgb=True)
    net_train = vgg16_convs(num_classes=C, device=cuda, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False, is_train=True)
    with pytest.raises(ValueError, match="is_train"):
        net_train.forward(data, meta, ext, estimate_rgb=True)
    with pytest.raises(ValueError, match="estimate_depth"):
        net.forward(data, meta, ext, dense_vertex=False, refine_depth=depth, refine_points=pts)
