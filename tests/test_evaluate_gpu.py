"""The device evaluator (posecnn_b200/evaluate.py, csrc/evaluate.cu, DESIGN.md §14) against the goldens made with the reference's
own pose_error.py and against the oracle tests/eval_ref.py: histogram exact, per-pair errors to 1e-6 deg / 1e-9 m / 1e-6 m /
1e-3 px, counts exact except pairs within those tolerances of their threshold (reported as ambiguous)."""
import os

import numpy as np
import pytest
import torch

from posecnn_b200 import synth
from posecnn_b200.evaluate import LOV_EVAL_SYMMETRIC, Evaluator, gt_rows_from_pose_blob
from tests import eval_ref

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "eval.npz"))
SETS = ("poses", "poses_refined", "poses_icp")
TOL = (1e-6, 1e-9, 1e-6, 1e-3)       # re deg, te m, ADD / ADD-S m, reproj px


def case(tag):
    return {k[len(tag) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(tag + "_")}


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def device_pairs(out):
    n = int(out["num_pairs"].item())
    return out["pairs"][:n].cpu().numpy(), out["errors"][:, :n].cpu().numpy(), out["flags"][:, :n].cpu().numpy()


def check_errors(errors, flags, ref_errors, ref_flags, thr_pairs):
    """Tolerances of the module docstring; re also passes when the two cosines agree to 4e-15 (acos is ill-conditioned at 0 and
    180 degrees).  Returns the number of ambiguous (pair, set) entries: within tolerance of the ADD / 5 px / 90 degree thresholds."""
    assert errors.shape == ref_errors.shape
    d = np.abs(errors - ref_errors)
    cos_ok = np.abs(np.cos(np.radians(errors[..., 0])) - np.cos(np.radians(ref_errors[..., 0]))) <= 4e-15
    assert ((d[..., 0] <= TOL[0]) | cos_ok).all(), d[..., 0].max()
    for i in (1, 2, 3):
        assert (d[..., i] <= TOL[i]).all(), (i, d[..., i].max())
    amb = (np.abs(ref_errors[..., 2] - thr_pairs) <= TOL[2]) | (np.abs(ref_errors[..., 3] - 5.0) <= TOL[3]) | \
          (np.abs(ref_errors[..., 0] - 90.0) <= TOL[0])
    assert (flags[~amb] == ref_flags[~amb]).all()
    if amb.any():
        print("ambiguous (pair, set) entries:", int(amb.sum()))
    return int(amb.sum())


def check_counts(got, want, ambiguous):
    diff = np.abs(np.asarray(got, np.int64) - np.asarray(want, np.int64))
    assert (diff[:, 0] == 0).all() and diff.sum() <= ambiguous, diff


def make_labels(B, H, W, C, seed, p_noise=0.05):
    """Label maps of the shape the network writes: coherent blocks (~75 % background), a few noisy pixels, gt -1 borders."""
    rng = np.random.default_rng(seed)
    gt = np.zeros((B, H, W), np.int32)
    for b in range(B):
        for _ in range(5):
            y, x = rng.integers(0, H - 60), rng.integers(0, W - 80)
            gt[b, y:y + rng.integers(20, 120), x:x + rng.integers(20, 160)] = rng.integers(1, C)
    gt[:, :, :3] = -1
    pred = np.where(rng.random((B, H, W)) < p_noise, rng.integers(0, C, (B, H, W)), np.maximum(gt, 0)).astype(np.int32)
    shift = np.roll(pred, 4, axis=2)
    return gt, np.where(rng.random((B, H, W)) < 0.5, pred, shift).astype(np.int32)


def evaluator(c, dev, sets=SETS, P=2620):
    C = int(c["C"])
    return Evaluator(C, synth.make_model_points(C, P), c["extents"], c["symmetric"], flip_z=c["flip_z"], pose_sets=sets, device=dev)


def score_case(ev, c, dev):
    out = ev.add_poses(T(c["gt_rows"], dev), T(c["rois"], dev), {s: T(c["poses"][i], dev) for i, s in enumerate(SETS)},
                       torch.tensor([int(c["num_rows"])], dtype=torch.int32, device=dev), T(c["meta"], dev))
    ev.add_labels(T(c["gt_label"], dev), T(c["label"], dev))
    return out


@pytest.mark.parametrize("C", [22, 2])
def test_confusion_exact_full_batch(cuda, C):
    gt, pred = make_labels(32, 480, 640, C, seed=C)
    ev = Evaluator(C, np.zeros((C, 1, 3)), np.ones((C, 3)), np.zeros(C), device=cuda)
    ev.add_labels(T(gt, cuda), T(pred, cuda))
    want = eval_ref.fast_hist(gt.reshape(-1), pred.reshape(-1), C)
    np.testing.assert_array_equal(ev.hist.cpu().numpy(), want)
    # an odd pixel count and an unaligned start take the scalar path: the same counts
    ev2 = Evaluator(C, np.zeros((C, 1, 3)), np.ones((C, 3)), np.zeros(C), device=cuda)
    g, p = T(gt, cuda).reshape(-1)[1:], T(pred, cuda).reshape(-1)[1:]
    ev2.add_labels(g, p)
    np.testing.assert_array_equal(ev2.hist.cpu().numpy(), eval_ref.fast_hist(gt.reshape(-1)[1:], pred.reshape(-1)[1:], C))
    s, r = ev.summary(), eval_ref.summary(want, np.zeros((1, 3, C), np.int64), ["poses"])
    for k in ("overall_accuracy", "mean_accuracy", "mean_iu", "fwavacc"):
        assert s[k] == pytest.approx(r[k], rel=1e-15, abs=0), k
    np.testing.assert_array_equal(s["per_class_iu"], r["per_class_iu"])


def test_prediction_out_of_range_is_reported(cuda):
    ev = Evaluator(4, np.zeros((4, 1, 3)), np.ones((4, 3)), np.zeros(4), device=cuda)
    gt = torch.zeros((1, 8, 8), dtype=torch.int32, device=cuda)
    pred = gt.clone()
    pred[0, 2, 3] = 4
    pred[0, 5, 5] = -2
    ev.add_labels(gt, pred)
    assert int(ev.hist.sum()) == 62 and int(ev.status[0]) == 2
    with pytest.raises(ValueError, match="2 predicted labels"):
        ev.summary()


@pytest.mark.parametrize("tag", eval_ref.CASES)
def test_pose_errors_match_goldens_and_oracle(cuda, tag):
    c = case(tag)
    C = int(c["C"])
    ev = evaluator(c, cuda)
    pairs, errors, flags = device_pairs(score_case(ev, c, cuda))
    np.testing.assert_array_equal(pairs, c["pairs"])
    thr = c["threshold"][c["gt_rows"][pairs[:, 0], 1].astype(int)].astype(np.float64)
    amb = check_errors(errors, flags, c["errors"], c["flags"], thr)
    check_counts(ev.counts.cpu().numpy(), c["counts"], amb)
    np.testing.assert_array_equal(ev.hist.cpu().numpy(), c["hist"])
    r = eval_ref.score(c["gt_rows"], c["rois"], list(c["poses"]), int(c["num_rows"]), c["meta"], synth.make_model_points(C, 2620),
                       c["symmetric"], c["threshold"], c["flip_z"], C)
    check_errors(errors, flags, r[1], r[2], thr)
    s = ev.summary()
    for i, name in enumerate(SETS):
        np.testing.assert_array_equal(s["poses"][name]["count_all"], c["counts"][i, 0])
        a = s["poses"][name]["accuracy"]
        assert np.isnan(a[c["counts"][i, 0] == 0]).all()


def test_deterministic_merge_and_graph_replay(cuda):
    c = case("lov")
    ev1, ev2 = evaluator(c, cuda), evaluator(c, cuda)
    o1, o2 = score_case(ev1, c, cuda), score_case(ev2, c, cuda)
    for k in ("pairs", "errors", "flags", "num_pairs"):
        n = int(o1["num_pairs"].item())
        a, b = (o1[k][:n], o2[k][:n]) if k == "pairs" else (o1[k], o2[k]) if k == "num_pairs" else (o1[k][:, :n], o2[k][:, :n])
        assert torch.equal(a, b), k
    assert torch.equal(ev1.state, ev2.state)
    # shard invariance: two evaluators over the two images (global image indices, batch_offset) merged == one over the batch
    halves = [evaluator(c, cuda) for _ in range(2)]
    for b, ev in enumerate(halves):
        sel = c["gt_rows"][:, 0] == b
        ev.add_poses(T(c["gt_rows"][sel], cuda), T(c["rois"], cuda), {s: T(c["poses"][i], cuda) for i, s in enumerate(SETS)},
                     torch.tensor([int(c["num_rows"])], dtype=torch.int32, device=cuda), T(c["meta"][b:b + 1], cuda), batch_offset=b)
        ev.add_labels(T(c["gt_label"][b:b + 1], cuda), T(c["label"][b:b + 1], cuda))
    halves[0].merge(halves[1])
    assert torch.equal(halves[0].state, ev1.state)
    # one add_labels + add_poses captured in a CUDA graph, replayed twice: twice the counts
    ev = evaluator(c, cuda)
    args = (T(c["gt_rows"], cuda), T(c["rois"], cuda), {s: T(c["poses"][i], cuda) for i, s in enumerate(SETS)},
            torch.tensor([int(c["num_rows"])], dtype=torch.int32, device=cuda), T(c["meta"], cuda))
    gl, lb = T(c["gt_label"], cuda), T(c["label"], cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ev.add_poses(*args)                  # warm-up outside the capture
        ev.add_labels(gl, lb)
    torch.cuda.current_stream().wait_stream(s)
    ev.state.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ev.add_poses(*args)
        ev.add_labels(gl, lb)
    assert not ev.state.any()                # capture runs nothing
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(ev.state, 2 * ev1.state)
    n = int(o1["num_pairs"].item())
    assert torch.equal(out["errors"][:, :n], o1["errors"][:, :n])


def test_gt_rows_from_pose_blob(cuda):
    rng = np.random.default_rng(4)
    blob = np.zeros((6, 13), np.float32)
    blob[:, 0] = [0, 0, 1, 1, 2, 2]
    blob[:, 1] = [1, 3, 2, 5, 4, 1]
    blob[:, 6:10] = rng.normal(size=(6, 4))
    blob[1, 6:10] = 0                        # the identity branch
    blob[:, 10:13] = rng.normal(size=(6, 3))
    rows = gt_rows_from_pose_blob(T(blob, cuda)).cpu().numpy()
    for i in range(6):
        RT = eval_ref.estimate_rt(np.r_[blob[i, 6:10], blob[i, 10:13]])
        np.testing.assert_array_equal(rows[i], np.r_[blob[i, :2], RT.reshape(-1)])


def scene_gt_rows(poses9):
    rows = np.zeros((poses9.shape[0], 14), np.float32)
    for i, r in enumerate(poses9):
        RT = np.zeros((3, 4), np.float32)
        RT[:, :3] = synth.quat_to_rot(r[2:6])
        RT[:, 3] = r[6:9]
        rows[i] = np.r_[r[0], r[1], RT.reshape(-1)]
    return rows


def compare_end_to_end(ev, calls, gt_rows, meta, pts, C, label_gt, label_pred):
    """calls: (rois, {set: poses}, num_rows) already scored by ev; eval_ref on the D2H copies must give the same figures."""
    want = np.zeros(ev.counts.shape, np.int64)
    amb = 0
    thr, sym, flip = ev.threshold.cpu().numpy(), ev.symmetric.cpu().numpy(), ev.flip_z.cpu().numpy()
    for (rois, sets, nr), out in calls:
        n = int(nr.item())
        names = list(sets)
        r = eval_ref.score(gt_rows, rois.cpu().numpy(), [sets[k].cpu().numpy() for k in names], n, meta, pts, sym, thr, flip, C)
        pairs, errors, flags = device_pairs(out)
        np.testing.assert_array_equal(pairs, r[0])
        t = thr[gt_rows[pairs[:, 0], 1].astype(int)].astype(np.float64)
        amb += check_errors(errors, flags, r[1], r[2], t)
        for i, k in enumerate(names):
            want[ev.pose_sets.index(k)] += r[3][i]
    check_counts(ev.counts.cpu().numpy(), want, amb)
    np.testing.assert_array_equal(ev.hist.cpu().numpy(), eval_ref.fast_hist(label_gt.reshape(-1), label_pred.reshape(-1), C))
    return want


def test_end_to_end_network_records(cuda):
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    C, B, H, W = 6, 2, 128, 160
    sc = synth.make_refine_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=3, seed=5, min_pixels=100)
    rgb, _ = synth.make_images(B, H, W, seed=3)
    meta, ext, pts = sc["meta"], synth.extents_for(C), sc["points"]
    gt_rows = scene_gt_rows(sc["poses"])
    dev = cuda
    # 2-D network with the ICP refinement
    net = vgg16_convs(num_classes=C, device=dev).init_random(seed=0, bias_std=0.05)
    L = net.forward(T(rgb, dev), T(meta, dev), T(ext, dev), sync_rois=False, refine_depth=T(sc["depth"], dev), refine_points=T(pts, dev))
    ev = Evaluator(C, pts, ext, np.r_[0, 0, 0, 1, 0, 0].astype(np.float32), pose_sets=SETS, device=dev)
    sets = {"poses": L["detections_poses"], "poses_refined": L["detections_poses_refined"], "poses_icp": L["detections_poses_icp"]}
    out = ev.add_poses(T(gt_rows, dev), L["detections_rois"], sets, L["num_detections"], T(meta, dev))
    ev.add_labels(T(sc["label"], dev), L["label_2d"])
    want = compare_end_to_end(ev, [((L["detections_rois"], sets, L["num_detections"]), out)], gt_rows, meta, pts, C, sc["label"],
                              L["label_2d"].cpu().numpy())
    assert want[0, 0].sum() == gt_rows.shape[0]
    # object-coordinate network: the depth estimate, its refinement, and the colour-only records as a fourth set
    cs = synth.make_coordinate_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=3, seed=6)
    gt3 = scene_gt_rows(cs["poses"])
    net3 = vgg16_convs(num_classes=C, device=dev, vertex_reg_2d=False, vertex_reg_3d=True, pose_reg=False).init_random(seed=0, bias_std=0.05)
    keys = torch.tensor([3, 9], dtype=torch.int64, device=dev)
    depth = T(cs["depth"], dev)
    L3 = net3.forward(T(rgb, dev), T(cs["meta"], dev), T(ext, dev), dense_vertex=False, estimate_keys=keys, estimate_rgb=True,
                      estimate_depth=depth, refine_depth=depth, refine_points=T(pts, dev))
    ev3 = Evaluator(C, pts, ext, np.zeros(C), pose_sets=SETS + ("poses_rgb",), device=dev)
    s3 = {"poses": L3["detections_poses"], "poses_refined": L3["detections_poses_refined"], "poses_icp": L3["detections_poses_icp"]}
    o3 = ev3.add_poses(T(gt3, dev), L3["detections_rois"], s3, L3["num_detections"], T(cs["meta"], dev))
    srgb = {"poses_rgb": L3["detections_poses_rgb"]}
    orgb = ev3.add_poses(T(gt3, dev), L3["detections_rois_rgb"], srgb, L3["num_detections_rgb"], T(cs["meta"], dev))
    ev3.add_labels(T(cs["label"], dev), L3["label_2d"])
    compare_end_to_end(ev3, [((L3["detections_rois"], s3, L3["num_detections"]), o3),
                             ((L3["detections_rois_rgb"], srgb, L3["num_detections_rgb"]), orgb)],
                       gt3, cs["meta"], pts, C, cs["label"], L3["label_2d"].cpu().numpy())
    s = ev3.summary()
    assert set(s["poses"]) == set(SETS + ("poses_rgb",))


def test_lov_symmetric_table_drives_adds(cuda):
    """A symmetric class is scored with ADD-S: for an estimate rotated about the ellipsoid's axis ADD-S is well below ADD."""
    C = 22
    c = dict(C=C, extents=synth.extents_for(C), flip_z=np.zeros(C, np.float32))
    rows = np.zeros((1, 14), np.float32)
    rows[0, :2] = (0, 13)
    rows[0, 2:] = np.c_[np.eye(3), [0, 0, 1.0]].reshape(-1)
    rois = np.zeros((1, 7), np.float32)
    rois[0, :2] = (0, 13)
    pose = np.array([[np.cos(0.5), 0, 0, np.sin(0.5), 0, 0, 1.0]], np.float32)
    got = {}
    for name, sym in (("adds", LOV_EVAL_SYMMETRIC), ("add", np.zeros(C, np.float32))):
        ev = evaluator(dict(c, symmetric=sym), cuda, sets=("poses",))
        out = ev.add_poses(T(rows, cuda), T(rois, cuda), {"poses": T(pose, cuda)}, None, T(synth.make_meta(synth.intrinsics())[None], cuda))
        got[name] = float(out["errors"][0, 0, 2])
    assert got["adds"] < 0.5 * got["add"]
