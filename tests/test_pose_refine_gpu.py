"""Pose refinement on the GPU (csrc/pose_refine.cu) against the float64 restatement tests/pose_refine_ref.py: every Gauss-Newton
step of every hypothesis, the chosen hypothesis and the final poses; planted recovery; determinism, graph capture, shards; the
network's refine_depth path and the synthesizer-style Refiner.  Measured deltas are printed (DESIGN.md §12 records them)."""
import numpy as np
import pytest
import torch

from posecnn_b200 import synth
from posecnn_b200.pose_refine import Refiner, refine_poses
from tests import pose_refine_ref as ref
from tests.test_pose_refine_cpu import PLANTED_ROT_DEG, PLANTED_SEEDS, PLANTED_TRANS_M, observable_rot_err_deg, planted_cases, rot_err_deg

pytestmark = pytest.mark.gpu
STEP_ROT, STEP_TRANS = 1e-4, 1e-4         # rad, m
FINAL_ROT, FINAL_TRANS = 1e-3, 5e-4


def make_case(B, C, seed, height=480, width=640):
    """Scene (3 objects per image at C = 22, one class-1 object per image at C = 2), ROI / pose rows (perturbed planted poses, plus a
    background row and an out-of-range class row) and the points table."""
    sc = synth.make_refine_scene(batch=B, height=height, width=width, num_classes=C, objects_per_image=3, seed=seed, noise_m=0.001)
    rng = np.random.default_rng(seed)
    rois, poses = [], []
    for row in sc["poses"]:
        qp, tp = synth.perturb_pose(row[2:6], row[6:9], rng)
        rois.append([row[0], row[1], 0, 0, 1, 1, 1.0])
        poses.append(np.r_[qp, tp])
    rois += [[0, 0, 0, 0, 1, 1, 1.0], [0, C, 0, 0, 1, 1, 1.0]]
    poses += [poses[0], poses[0]]
    return dict(label=sc["label"], depth=sc["depth"], meta=sc["meta"], rois=np.array(rois, np.float32),
                poses=np.array(poses, np.float32), points=sc["points"])


def to_dev(case, cuda):
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return {k: T(v) for k, v in case.items()}


def check_against_oracle(case, out, batch_offset=0, iterations=8):
    label, depth, meta, rois, poses, pts = (case[k] for k in ("label", "depth", "meta", "rois", "poses", "points"))
    tr = out["icp_trace"].cpu().numpy().astype(np.float64)
    info = out["icp_info"].cpu().numpy()
    want = ref.refine(label, depth, meta, rois, poses, pts, batch_offset=batch_offset, iterations=iterations)
    np.testing.assert_allclose(out["poses_refined"].cpu().numpy(), want["poses_refined"], rtol=1e-5, atol=1e-6)
    worst = dict(steps=0, step_rot=0.0, step_trans=0.0, inl=0, final_rot=0.0, final_trans=0.0, same_h=0, rows=0)
    P = pts.shape[1]
    for r in range(rois.shape[0]):
        np.testing.assert_array_equal(info[r, 0], want["icp_info"][r, 0])
        if want["icp_info"][r, 2] == 0 and not want["poses_icp"][r].any():
            assert not out["poses_icp"][r].any() and not tr[r].any()
            continue
        worst["rows"] += 1
        b, c = int(rois[r, 0]) - batch_offset, int(rois[r, 1])
        m = meta.reshape(label.shape[0], -1)[b].astype(np.float64)
        live = ref.Live(label[b], depth[b], c, m[0], m[4], m[2], m[5], 10000.0, 0.25, 6.0)
        scores = []
        for h in range(ref.NUM_HYP):
            for s in range(iterations):
                q, t, n_gpu = tr[r, h, s, :4], tr[r, h, s, 4:7], tr[r, h, s, 7]
                a = ref.associate(live, pts[c], q, t, 0.01)
                near = ref.near_gate_count(live, a, 0.01)
                assert abs(int(a["inlier"].sum()) - n_gpu) <= near, (r, h, s, a["inlier"].sum(), n_gpu, near)
                worst["inl"] = max(worst["inl"], abs(int(a["inlier"].sum()) - int(n_gpu)))
                qn, tn, _, stop = ref.gn_step(live, pts[c], q, t, 0.01)
                nxt = tr[r, h, s + 1]
                if int(a["inlier"].sum()) != n_gpu:     # a point at a gate went the other way: another system, not comparable
                    continue
                worst["steps"] += 1
                if stop:
                    np.testing.assert_array_equal(nxt[:7], tr[r, h, s, :7])
                    continue
                dr, dt = np.radians(rot_err_deg(qn, nxt[:4])), np.linalg.norm(tn - nxt[4:7])
                assert dr <= STEP_ROT and dt <= STEP_TRANS, (r, h, s, dr, dt)
                worst["step_rot"], worst["step_trans"] = max(worst["step_rot"], dr), max(worst["step_trans"], dt)
            scores.append(ref.score(live, pts[c], want["icp_trace"][r, h, -1, :4], want["icp_trace"][r, h, -1, 4:7])[0])
        srt = sorted(scores, reverse=True)
        if srt[0] - srt[1] >= 3 or srt[0] == srt[1] == scores[0]:
            assert info[r, 1] == want["icp_info"][r, 1], (r, scores, info[r])
        if info[r, 1] == want["icp_info"][r, 1]:
            worst["same_h"] += 1
            g, w = out["poses_icp"][r].cpu().numpy(), want["poses_icp"][r]
            dr, dt = np.radians(rot_err_deg(g[:4], w[:4])), np.linalg.norm(g[4:] - w[4:])
            assert dr <= FINAL_ROT and dt <= FINAL_TRANS, (r, dr, dt)
            worst["final_rot"], worst["final_trans"] = max(worst["final_rot"], dr), max(worst["final_trans"], dt)
    print("oracle deltas:", worst, "P =", P)
    assert worst["rows"] >= 2


@pytest.mark.parametrize("B,C", [(2, 22), (4, 2)])
def test_against_oracle_per_step(cuda, B, C):
    case = make_case(B, C, seed=11 + B)
    d = to_dev(case, cuda)
    num = torch.tensor([case["rois"].shape[0]], dtype=torch.int32, device=cuda)
    out = refine_poses(d["label"], d["depth"], d["meta"], d["rois"], d["poses"], d["points"], num_rows=num, trace=True)
    check_against_oracle(case, out)


def test_shard_batch_offset_against_oracle(cuda):
    case = make_case(4, 22, seed=21)
    d = to_dev(case, cuda)
    full = refine_poses(d["label"], d["depth"], d["meta"], d["rois"], d["poses"], d["points"], trace=True)
    sel = np.where(case["rois"][:, 0] >= 2)[0]
    shard = dict(case, label=case["label"][2:], depth=case["depth"][2:], meta=case["meta"][2:], rois=case["rois"][sel],
                 poses=case["poses"][sel])
    ds = to_dev(shard, cuda)
    part = refine_poses(ds["label"], ds["depth"], ds["meta"], ds["rois"], ds["poses"], ds["points"], batch_offset=2, trace=True)
    for k in ("poses_refined", "poses_icp", "icp_info", "icp_trace"):
        assert torch.equal(part[k], full[k][torch.from_numpy(sel).to(cuda)]), k
    check_against_oracle(shard, part, batch_offset=2)


@pytest.mark.parametrize("seed", PLANTED_SEEDS)
def test_planted_recovery_on_device(cuda, seed):
    """Every object of the scene in one batched call, with the full point table, to the CPU test's bounds."""
    cases = planted_cases(seed)
    sc = cases[0][0]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rois = np.stack([c[1] for c in cases]).astype(np.float32)
    poses = np.stack([c[2] for c in cases]).astype(np.float32)
    out = refine_poses(T(sc["label"]), T(sc["depth"]), T(sc["meta"]), T(rois), T(poses), T(sc["points"]))
    ext = synth.extents_for(22)
    for r, (_, roi, _, gt) in enumerate(cases):
        icp = out["poses_icp"][r].cpu().numpy().astype(np.float64)
        c = int(roi[1])
        er, et = observable_rot_err_deg(icp[:4], gt[:4], ext[c]), np.linalg.norm(icp[4:] - gt[4:])
        print("planted class", c, "rot err deg", er, "trans err m", et)
        assert er < PLANTED_ROT_DEG and et < PLANTED_TRANS_M, c


def test_determinism_graph_capture_and_num_rows(cuda):
    case = make_case(2, 22, seed=13)
    d = to_dev(case, cuda)
    cap = case["rois"].shape[0]
    num = torch.tensor([cap - 2], dtype=torch.int32, device=cuda)
    args = (d["label"], d["depth"], d["meta"], d["rois"], d["poses"], d["points"])
    a = refine_poses(*args, num_rows=num, trace=True)
    b = refine_poses(*args, num_rows=num, trace=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for k in ("poses_refined", "poses_icp", "icp_info", "icp_trace"):
        assert not a[k][cap - 2:].any(), k          # rows past num_rows
    assert a["poses_icp"][: cap - 2].abs().sum(1).gt(0).sum() >= 2
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        refine_poses(*args, num_rows=num, trace=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = refine_poses(*args, num_rows=num, trace=True)
    num.fill_(cap)
    g.replay()
    full = refine_poses(*args, trace=True)
    for k in a:
        assert torch.equal(c[k], full[k]), k


def test_refiner_icp_python_matches_batched_rows(cuda):
    case = make_case(2, 22, seed=17)
    d = to_dev(case, cuda)
    out = refine_poses(d["label"], d["depth"], d["meta"], d["rois"], d["poses"], d["points"])
    sel = np.where(case["rois"][:, 0] == 1)[0]
    K = case["meta"][1, :9].reshape(3, 3)
    from posecnn_b200.utils.results import icp_parameters
    prm = icp_parameters(K, 10000.0)
    n = len(sel)
    o1, o2 = np.zeros((n, 7), np.float32), np.zeros((n, 7), np.float32)
    Refiner(case["points"], device=cuda).icp_python(case["label"][1], case["depth"][1], prm, 480, 640, n, 7, case["rois"][sel],
                                                    case["poses"][sel], o1, o2, 0.01)
    np.testing.assert_array_equal(o1, out["poses_refined"][sel].cpu().numpy())
    np.testing.assert_array_equal(o2, out["poses_icp"][sel].cpu().numpy())


def test_invalid_arguments_raise(cuda):
    case = make_case(2, 22, seed=13)
    d = to_dev(case, cuda)
    big = torch.zeros((22, 4097, 3), device=cuda)
    with pytest.raises(RuntimeError, match="P = 4097"):
        refine_poses(d["label"], d["depth"], d["meta"], d["rois"], d["poses"], big)
    with pytest.raises(RuntimeError, match="znear < zfar"):
        refine_poses(d["label"], d["depth"], d["meta"], d["rois"], d["poses"], d["points"], znear=6.0, zfar=1.0)
    with pytest.raises(RuntimeError, match="iterations"):
        refine_poses(d["label"], d["depth"], d["meta"], d["rois"], d["poses"], d["points"], iterations=-1)


def test_network_refine_depth_eager_graph_and_off(cuda):
    from posecnn_b200.networks.vgg16_convs import GraphedForward, vgg16_convs
    C, B, H, W = 6, 2, 128, 160
    net = vgg16_convs(num_classes=C, device=cuda).init_random(seed=0, bias_std=0.05)
    rgb, depth_m = synth.make_images(B, H, W, seed=3)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    data, meta, ext = T(rgb), T(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)), T(synth.extents_for(C))
    depth = T((depth_m * 10000.0).astype(np.float32))
    pts = T(synth.make_model_points(C, 500))
    off = {k: v.clone() for k, v in net.forward(data, meta, ext, sync_rois=False).items()}
    on = {k: v.clone() for k, v in net.forward(data, meta, ext, sync_rois=False, refine_depth=depth, refine_points=pts).items()}
    new = {"detections_poses_refined", "detections_poses_icp", "detections_icp_info"}
    assert set(on) - set(off) == new and set(off) <= set(on)
    for k in off:
        assert torch.equal(off[k], on[k]), k
    n = int(on["num_detections"].item())
    assert n >= 1 and not on["detections_poses_icp"][n:].any()
    assert on["detections_icp_info"][:n, 0].gt(0).any()
    gf = GraphedForward(net, data, meta, ext, refine_depth=depth, refine_points=pts)
    L = gf(data, meta, refine_depth=depth)
    torch.cuda.synchronize()
    for k in new | {"detections_rois", "detections_poses"}:
        assert torch.equal(L[k], on[k]), k
    net_nopose = vgg16_convs(num_classes=C, device=cuda, pose_reg=False).init_random(seed=0)
    with pytest.raises(ValueError, match="pose_reg"):
        net_nopose.forward(data, meta, ext, refine_depth=depth, refine_points=pts)
    gf0 = GraphedForward(net, data, meta, ext)
    L0 = gf0(data, meta)
    assert not (set(L0) & new)
