"""Object-coordinate pose estimation on the GPU (csrc/coord_pose.cu, DESIGN.md §13) against the float64 restatement
tests/coord_pose_ref.py on analytic 480x640 scenes: hypotheses (class, attempts, pixel triple) and per-round subsets exactly, counts
and survivors, final poses; planted recovery; dense and low-resolution sources bit-identical; shards, determinism, CUDA-graph
replay; edge cases; the synthesizer-style wrapper.  Measured deltas are printed (DESIGN.md §13 records them)."""
import numpy as np
import pytest
import torch

from posecnn_b200 import heads, synth
from posecnn_b200.coord_pose import CoordPoseEstimator, estimate_poses_3d
from tests import coord_pose_ref as ref
from tests.test_coord_pose_cpu import PLANTED_ROT_DEG, PLANTED_TRANS_M, rot_err_deg

pytestmark = pytest.mark.gpu
KEYS = [0x1234567890ABCDEF, 77, 2**63 + 5, 31337]


def scene(B, C, seed, noise=0.0, outliers=0.0):
    return synth.make_coordinate_scene(batch=B, num_classes=C, objects_per_image=3 if C > 2 else 1, seed=seed, coord_noise_m=noise,
                                       outlier_fraction=outliers)


def run(sc, cuda, keys, trace=False, **kw):
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    B = sc["label"].shape[0]
    k = torch.tensor(np.array(keys[:B], np.uint64).view(np.int64), device=cuda)
    src = kw.pop("src", None) or dict(vertex=T(sc["vertex"]))
    return estimate_poses_3d(T(sc["label"]), T(sc["depth"]), T(sc["meta"]), T(sc["extents"]), k, trace=trace, **src, **kw)


def host(out):
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("B,C,noise,outliers,seed", [(1, 22, 0.0, 0.0, 3), (2, 22, 0.002, 0.2, 4), (1, 2, 0.0, 0.2, 5),
                                                     (4, 2, 0.002, 0.0, 6)])
def test_against_oracle(cuda, B, C, noise, outliers, seed):
    sc = scene(B, C, seed, noise, outliers)
    out = host(run(sc, cuda, KEYS, trace=True))
    worst = dict(rot=0.0, trans=0.0, count=0, objects=0)
    for b in range(B):
        cam = (sc["meta"][b, 0], sc["meta"][b, 4], sc["meta"][b, 2], sc["meta"][b, 5])
        want = ref.estimate_image(sc["label"][b], sc["depth"][b], sc["vertex"][b], sc["extents"], cam, 10000.0, KEYS[b], C)
        th = out["trace_hyp"][b]
        for h, hy in enumerate(want["hyps"]):          # drawn objects and pixel triples: exact
            assert (th[h, 0], th[h, 1]) == (hy["obj"], hy["attempts"]), (b, h)
            assert list(th[h, 2:5]) == (hy["pix"] if hy["obj"] else [-1, -1, -1]), (b, h)
        np.testing.assert_array_equal(out["info"][b][:, [0, 1, 4]], want["info"][:, [0, 1, 4]])
        for c, rounds in want["rounds"].items():
            worst["objects"] += 1
            tr = out["trace_round"][b, c]
            for r, rd in enumerate(rounds):              # subsets: exact
                assert tr[r, 0] == rd["taken"] and (int(tr[r, 1]) & 0xFFFFFFFF) == rd["hash"], (b, c, r)
                worst["count"] = max(worst["count"], abs(int(tr[r, 3]) - rd["best_count"]))
            assert out["info"][b, c, 5] == want["info"][c, 5], (b, c)        # survivor
            worst["rot"] = max(worst["rot"], rot_err_deg(out["poses"][b, c, :, :3].astype(np.float64), want["poses"][c, :, :3]))
            worst["trans"] = max(worst["trans"], float(np.linalg.norm(out["poses"][b, c, :, 3] - want["poses"][c, :, 3])))
    print(f"\n[coord_pose oracle] B={B} C={C} noise={noise} outliers={outliers}: {worst}")
    assert worst["count"] <= 2 and worst["rot"] < 0.05 and worst["trans"] < 5e-4 and worst["objects"] >= 1


def test_planted_recovery(cuda):
    sc = scene(4, 22, 11)
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
    print(f"\n[coord_pose planted] {n} objects: worst {worst_r:.4f} deg, {1000 * worst_t:.3f} mm")
    assert n >= 6 and worst_r < PLANTED_ROT_DEG and worst_t < PLANTED_TRANS_M


def test_lowres_source_bit_identical_to_dense(cuda):
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
    part = {k: sc[k][2:4] for k in ("label", "depth", "meta", "vertex")}
    part["extents"] = sc["extents"]
    shard = run(part, cuda, KEYS[2:], trace=True)
    for k in whole:
        assert torch.equal(whole[k][2:4], shard[k]), k
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    inp = dict(label=T(sc["label"]), depth=T(sc["depth"]), meta=T(sc["meta"]), ext=T(sc["extents"]), vertex=T(sc["vertex"]),
               keys=torch.tensor(np.array(KEYS, np.uint64).view(np.int64), device=cuda))
    f = lambda: estimate_poses_3d(inp["label"], inp["depth"], inp["meta"], inp["ext"], inp["keys"], vertex=inp["vertex"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = f()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(res["poses"], whole["poses"]) and torch.equal(res["info"], whole["info"])


def test_edge_cases_give_zero_rows(cuda):
    C = 6
    sc = scene(2, C, 19)
    sc["depth"][1] = 0.0                                          # image 1: every pixel a hole
    small = int(sc["poses"][0, 1])
    keep = np.argwhere(sc["label"][0] == small)[:300]
    sc["label"][0][sc["label"][0] == small] = 0
    sc["label"][0][keep[:, 0], keep[:, 1]] = small                # <= 400 pixels
    zero_c = [int(r[1]) for r in sc["poses"] if r[0] == 0 and int(r[1]) != small and (sc["label"][0] == int(r[1])).sum() > 400]
    assert zero_c, "the scene must hold a second object for the zero-extents case"
    sc["extents"] = sc["extents"].copy()
    for c in zero_c[:1]:
        sc["extents"][c] = 0.0
    out = host(run(sc, cuda, KEYS))
    assert not out["poses"][1].any()
    assert (out["info"][1, 1:, 4] == 256).all()                  # every hypothesis of image 1 hit the attempt cap
    assert not out["poses"][0, small].any() and out["info"][0, small, 0] <= 400
    for c in zero_c[:1]:
        assert not out["poses"][0, c].any() and out["info"][0, c, 1] == 0
    absent = [c for c in range(1, C) if not (sc["label"][0] == c).any()]
    for c in absent:
        assert not out["poses"][0, c].any() and out["info"][0, c, 5] == -1


def test_wrapper_equals_batched_rows(cuda):
    C = 22
    sc = scene(1, C, 23, 0.002, 0.2)
    out = host(run(sc, cuda, KEYS))
    poses = np.zeros((3, 4, C), np.float32)
    m = sc["meta"][0]
    CoordPoseEstimator(key=KEYS[0]).estimate_poses_3d(sc["label"][0], sc["depth"][0], sc["vertex"][0], sc["extents"],
                                                      poses, C, m[0], m[4], m[2], m[5], 10000.0)
    np.testing.assert_array_equal(poses, out["poses"][0].transpose(1, 2, 0))


def test_per_hypothesis_counts_against_oracle(cuda):
    """Every hypothesis's inlier count in every round, within the number of its pairs whose distance lies within 1e-6 relative
    of the 1 cm gate (the only pairs a last-bit difference of the pose can move across it)."""
    B, C = 1, 22
    sc = scene(B, C, 29, 0.002, 0.2)
    out = host(run(sc, cuda, KEYS, trace=True))
    cam = (sc["meta"][0, 0], sc["meta"][0, 4], sc["meta"][0, 2], sc["meta"][0, 5])
    want = ref.estimate_image(sc["label"][0], sc["depth"][0], sc["vertex"][0], sc["extents"], cam, 10000.0, KEYS[0], C)
    th = out["trace_hyp"][0]
    compared = 0
    for c, rounds in want["rounds"].items():
        for r, rd in enumerate(rounds):
            for h, n in rd["counts"].items():
                assert abs(int(th[h, 5 + r]) - n) <= rd["near"][h], (c, r, h)
                compared += 1
    counted = {(h, r) for rounds in want["rounds"].values() for r, rd in enumerate(rounds) for h in rd["counts"]}
    for h in range(ref.NUM_HYP):
        for r in range(ref.ROUNDS):
            if (h, r) not in counted:
                assert th[h, 5 + r] == -1
    assert compared >= 256


def test_records_equal_the_reference(cuda):
    from posecnn_b200.coord_pose import assemble_records
    from tests.test_coord_pose_cpu import golden_record_cases
    K, cases = golden_record_cases()
    for P, scale, rois, poses in cases:
        C = P.shape[2]
        meta = np.zeros((2, 48), np.float32)
        meta[:, :9] = (K * np.array([[scale, 1, scale], [1, scale, scale], [1, 1, 1]])).reshape(-1)
        meta[:, [1, 3, 6, 7]] = 0
        pt = torch.from_numpy(np.stack([P.transpose(2, 0, 1)] * 2)).to(cuda)          # two images, the second numbered 5 + 1
        r, p, n = assemble_records(pt, torch.from_numpy(synth.extents_for(C)).to(cuda), torch.from_numpy(meta).to(cuda), scale, 5)
        r, p, n = r.cpu().numpy(), p.cpu().numpy(), int(n.item())
        m = rois.shape[0]
        assert n == 2 * m and not r[n:].any() and not p[n:].any()
        for i in range(2):
            np.testing.assert_array_equal(r[i * m:(i + 1) * m, 0], 5 + i)
            np.testing.assert_array_equal(r[i * m:(i + 1) * m, 1], rois[:, 1])
            np.testing.assert_allclose(r[i * m:(i + 1) * m, 2:], rois[:, 2:], rtol=1e-5, atol=2e-3)
            np.testing.assert_allclose(p[i * m:(i + 1) * m], poses, rtol=0, atol=2e-6)


def test_network_estimate_depth_eager_graph_and_off(cuda):
    from posecnn_b200.coord_pose import assemble_records
    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    C, B, H, W = 6, 2, 128, 160
    net = vgg16_convs(num_classes=C, device=cuda, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False,
                      scales=(1.5,)).init_random(seed=0, bias_std=0.05)
    rgb, depth_m = synth.make_images(B, H, W, seed=3)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    data, meta, ext = T(rgb), T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)), T(synth.extents_for(C))
    depth = T((depth_m * 10000.0).astype(np.float32))
    keys = torch.tensor([3, 9], dtype=torch.int64, device=cuda)
    off = {k: v.clone() for k, v in net.forward(data, meta, ext, dense_vertex=False).items()}
    on = {k: v.clone() for k, v in net.forward(data, meta, ext, dense_vertex=False, estimate_depth=depth, estimate_keys=keys).items()}
    new = {"estimate_poses", "estimate_info", "detections_rois", "detections_poses", "num_detections"}
    assert set(on) - set(off) == new and set(off) <= set(on)
    for k in off:
        assert torch.equal(off[k], on[k]), k
    assert on["estimate_info"][..., 0].sum() > 0                     # the estimator ran on the network's own label maps
    est = estimate_poses_3d(on["label_2d"], depth, meta, ext, keys, lowres=net._last_lowres,
                            bias_vertex=net.params["vertex_pred/biases"])
    assert torch.equal(est["poses"], on["estimate_poses"])
    rr, pp, nn = assemble_records(est["poses"], ext, meta, 1.5, 0)
    assert torch.equal(rr, on["detections_rois"]) and torch.equal(pp, on["detections_poses"]) and torch.equal(nn, on["num_detections"])
    assert on["detections_rois"].shape == (B * (C - 1), 6)
    gf = GraphedForward(net, data, meta, ext, dense_vertex=False, estimate_depth=depth, estimate_keys=keys)
    L = gf(data, meta, estimate_depth=depth)
    torch.cuda.synchronize()
    for k in new:
        assert torch.equal(L[k], on[k]), k
    gf0 = GraphedForward(net, data, meta, ext, dense_vertex=False)
    L0 = gf0(data, meta)
    torch.cuda.synchronize()
    assert not (set(L0) & new)
    net2d = vgg16_convs(num_classes=C, device=cuda).init_random(seed=0)
    with pytest.raises(ValueError, match="vertex_reg_3d"):
        net2d.forward(data, meta, ext, estimate_depth=depth)
