"""The detection records on the device (det_records.detection_records, csrc/det.cu: k_det_records; DESIGN.md §16):

- seeded networks at 480 x 640, B = 32, C = 22 (A = 20) and C = 2 (A = 30), each also with every foreground logit dead so
  that the structural 1/C ties of cls_score's ReLU decide the top scores: selection exactly the restatement's (tests/det_post_ref.py), boxes within 2 ulp (expf against numpy's float32
  exp), translations and Nelder-Mead trace counts bit-exact against the restatement fed the device's own boxes;
- the reference's own post-processing (tests/golden/det_post.npz): the rule of tests/test_det_post_cpu.py;
- rows past num_rois are ignored and an image without proposals has no records;
- batch invariance, graph replay, sync_rois's class-ascending lists, and the C = 2 records scored through Evaluator (eggbox
  flip, ADD-S) equal to tests/eval_ref.py on the same records.
"""
import numpy as np
import pytest
import torch

from tests import det_post_ref as ref
from tests import eval_ref
from tests.test_det_post_cpu import case, compare_with_golden

pytestmark = pytest.mark.gpu

SCALES = {20: (4, 8, 16, 32), 30: (3, 4, 5, 6, 7, 8)}


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def images(B, seed):
    from posecnn_b200 import synth
    rgb, _ = synth.make_images(B, 480, 640, seed=seed)
    return torch.from_numpy(np.ascontiguousarray(rgb))


def metas(B):
    from posecnn_b200 import synth
    K = synth.intrinsics(480, 640)
    m = np.stack([synth.make_meta(K)] * B).astype(np.float32)
    m[1::2, 2] += np.float32(7.25)                    # two cameras
    return m


def network(dev, C, A, seed, P=2620, dead_foreground=False):
    """A seeded vgg16_det with the object-point table.  dead_foreground: every foreground cls_score bias is -10, so each
    foreground logit ReLUs to 0 and a row whose background logit does too has cls_prob exactly 1/C in every class: the top
    score of every class is then an exact tie between many rows.  At C = 2 the background bias is -10 too (the seeded
    network's background logit is positive on every row), so every row is such a tie."""
    from posecnn_b200 import synth
    from posecnn_b200.networks import vgg16_det
    net = vgg16_det(num_classes=C, anchor_scales=SCALES[A], device=dev).init_random(seed=seed, bias_std=0.05)
    if dead_foreground:
        net.params["cls_score/biases"][(1 if C > 2 else 0):] = -10.0
    return net.set_points(synth.make_model_points(C, P))


def host(L, *keys):
    return [L[k].cpu().numpy() for k in keys]


def check_against_restatement(L, meta, points, B, N, C):
    """Selection exact, boxes within 2 ulp, translations and trace counts bit-exact on the device's boxes.  Returns the
    number of (image, class) slots whose top score is an exact tie between rows."""
    cls_prob, bbox_pred, poses_tanh, rois, num = host(L, "cls_prob", "bbox_pred", "poses_tanh", "rois", "num_rois")
    dets, poses, num_dets, trace = host(L, "dets", "poses", "num_dets", "det_trace")
    boxes = ref.class_boxes(rois, ref.denormalise(bbox_pred), 480, 640)
    ties = 0
    for b in range(B):
        sel = dict(ref.select(cls_prob[b * N:(b + 1) * N], int(num[b])))
        assert int(num_dets[b]) == len(sel)
        K = meta[b, :9].astype(np.float64).reshape(3, 3)
        for j in range(1, C):
            slot = b * (C - 1) + j - 1
            if j not in sel:
                assert dets[slot, 0] == b and (dets[slot, 1:] == 0).all() and (poses[slot] == 0).all() and (trace[slot] == 0).all()
                continue
            row = b * N + sel[j]
            s = cls_prob[b * N:b * N + int(num[b]), j]
            ties += int((s == s.max()).sum() > 1)
            assert dets[slot, 0] == b and dets[slot, 1] == j and dets[slot, 6] == cls_prob[row, j]
            np.testing.assert_array_equal(poses[slot, :4], poses_tanh[row, 4 * j:4 * j + 4])   # the row, identified
            want = boxes[row, 4 * j:4 * j + 4]
            assert (np.abs(dets[slot, 2:6] - want) <= 2 * np.spacing(np.float32(1024))).all(), (b, j)
            t, srch = ref.translation(dets[slot, 2:6], poses[slot, :4], points[j], K)
            np.testing.assert_array_equal(poses[slot, 4:], t)
            assert tuple(trace[slot]) == (srch.nit, srch.nfev), (b, j)
    return ties


@pytest.mark.parametrize("C,A,dead", [(22, 20, False), (22, 20, True), (2, 30, False), (2, 30, True)])
def test_network_records_exact(cuda, C, A, dead):
    B, N = 32, 300
    net = network(cuda, C, A, seed=40 + C, dead_foreground=dead)
    meta = metas(B)
    L = net.forward(images(B, seed=C).to(cuda), sync_rois=False, meta_data=T(meta, cuda))
    ties = check_against_restatement(L, meta, net.points.cpu().numpy(), B, N, C)
    tr = L["det_trace"].cpu().numpy()
    filled = tr[:, 1] > 0
    print(f"C = {C}: {int(filled.sum())} records, {ties} with an exact tie at the top score; evaluations per record mean "
          f"{tr[filled, 1].mean():.1f}, max {tr[filled, 1].max()}")
    structural = int((L["cls_prob"].cpu().numpy() == np.float32(1) / np.float32(C)).all(1).sum())
    print(f"rows with every probability exactly 1/C: {structural}")
    if dead:
        assert structural > 0 and ties > 0                                    # exact 1/C ties deciding the top score


@pytest.mark.parametrize("tag", ["lov", "linemod"])
def test_records_against_reference(cuda, tag):
    from posecnn_b200.det_records import detection_records
    g = case(tag)
    dets, poses, num, trace = detection_records(T(g["cls_prob"], cuda), T(g["bbox_pred"], cuda), T(g["poses_tanh"], cuda),
                                                T(g["rois"], cuda), T(g["num_rois"], cuda), tuple(g["im_hw"]), T(g["meta"], cuda),
                                                T(g["points"], cuda))
    dets, poses, num, trace = (x.cpu().numpy() for x in (dets, poses, num, trace))
    filled = dets[:, 1] > 0
    assert int(num.sum()) == filled.sum() == g["ref_dets"].shape[0]
    d = dets[filled]
    assert (np.abs(d[:, 2:6] - g["ref_dets"][:, 2:6]) <= 2 * np.spacing(np.float32(1024))).all()
    same = (d[:, 2:6] == g["ref_dets"][:, 2:6]).all(1)
    print(f"{tag}: {int(same.sum())} / {same.size} boxes bit-equal to the reference's")
    n = compare_with_golden(tag, d, poses[filled], trace[filled], only=np.nonzero(same)[0])
    print(f"{tag}: {n} searches explained by decisions within the fp32 sensitivity")


def test_rows_past_num_rois_and_empty_images(cuda):
    from posecnn_b200.det_records import detection_records
    g = case("lov")
    B, N = g["num_rois"].shape[0], g["rois"].shape[0] // g["num_rois"].shape[0]
    args = lambda p, n: (T(p, cuda), T(g["bbox_pred"], cuda), T(g["poses_tanh"], cuda), T(g["rois"], cuda), T(n, cuda),
                         (480, 640), T(g["meta"], cuda), T(g["points"], cuda))
    base = [x.cpu().numpy() for x in detection_records(*args(g["cls_prob"], g["num_rois"]))]
    planted = g["cls_prob"].copy()
    planted[N + int(g["num_rois"][1]), 1:] = 1.0                              # the top score everywhere, in image 1's capacity row
    got = [x.cpu().numpy() for x in detection_records(*args(planted, g["num_rois"]))]
    for a, b in zip(base, got):
        np.testing.assert_array_equal(a, b)
    n = g["num_rois"].copy()
    n[1] = 0
    dets, poses, num, trace = (x.cpu().numpy() for x in detection_records(*args(g["cls_prob"], n)))
    C = g["cls_prob"].shape[1]
    assert num[1] == 0 and (dets[C - 1:, 1:] == 0).all() and (poses[C - 1:] == 0).all() and (dets[C - 1:, 0] == 1).all()
    np.testing.assert_array_equal(dets[:C - 1], base[0][:C - 1])
    assert num[0] == base[2][0]


def test_batch_invariance_and_graph_replay(cuda):
    from posecnn_b200.networks.vgg16_det import GraphedForward
    B = 4
    net = network(cuda, 22, 20, seed=9)
    data = images(B, seed=9).to(cuda)
    meta = T(metas(B), cuda)
    keys = ("dets", "poses", "num_dets", "det_trace")
    L = {k: v.clone() for k, v in net.forward(data, sync_rois=False, meta_data=meta).items()}
    S = 21
    for b in range(B):
        one = net.forward(data[b:b + 1].contiguous(), sync_rois=False, meta_data=meta[b:b + 1].contiguous())
        assert torch.equal(one["dets"][:, 1:], L["dets"][b * S:(b + 1) * S, 1:]), b
        for k in ("poses", "det_trace"):
            assert torch.equal(one[k], L[k][b * S:(b + 1) * S]), (b, k)
        assert torch.equal(one["num_dets"], L["num_dets"][b:b + 1])
    second = images(B, seed=10).to(cuda)
    meta2 = meta.clone()
    meta2[:, 2] += 5.0
    graphed = GraphedForward(net, data, meta_data=meta)
    got = {k: v.clone() for k, v in graphed(second, meta2).items()}
    torch.cuda.synchronize()
    want = net.forward(second, sync_rois=False, meta_data=meta2)
    for k in keys + ("cls_prob", "rois"):
        assert torch.equal(got[k], want[k]), k


def test_sync_rois_lists(cuda):
    net = network(cuda, 22, 20, seed=12)
    data = images(2, seed=12).to(cuda)
    meta = T(metas(2), cuda)
    full = {k: v.clone() for k, v in net.forward(data, sync_rois=False, meta_data=meta).items()}
    one = net.forward(data[:1].contiguous(), sync_rois=True, meta_data=meta[:1].contiguous())
    d = one["dets"].cpu().numpy()
    assert d.shape[0] == int(one["num_dets"][0]) and d.shape[1] == 7
    assert (d[:, 0] == 0).all() and (np.diff(d[:, 1]) > 0).all() and (d[:, 1] >= 1).all()   # the reference's rois [n,6]: d[:, 1:]
    fd, fp = full["dets"][:21].cpu().numpy(), full["poses"][:21].cpu().numpy()
    keep = fd[:, 1] > 0
    np.testing.assert_array_equal(d, fd[keep])
    np.testing.assert_array_equal(one["poses"].cpu().numpy(), fp[keep])
    two = net.forward(data, sync_rois=True, meta_data=meta)
    assert two["dets"].shape[0] == int(full["num_dets"].sum())


def test_linemod_records_scored_like_eval_ref(cuda):
    """C = 2 records straight into Evaluator.add_poses (empty slots are class 0 and pair with nothing), with LINEMOD's eggbox
    flip and ADD-S on the object, against tests/eval_ref.score on the same records."""
    from posecnn_b200 import synth
    from posecnn_b200.evaluate import Evaluator
    from tests.test_evaluate_gpu import check_counts, check_errors
    B, C = 8, 2
    net = network(cuda, C, 30, seed=77)
    meta = metas(B)
    L = net.forward(images(B, seed=77).to(cuda), sync_rois=False, meta_data=T(meta, cuda))
    dets, poses = L["dets"], L["poses"]
    rng = np.random.default_rng(77)
    gt = []
    for b in range(B):
        q = synth._rand_quat(rng)
        RT = np.zeros((3, 4), np.float32)
        RT[:, :3] = eval_ref.quat2mat(q)
        RT[:, 3] = (rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(0.5, 1.5))
        gt.append(np.r_[b, 1, RT.reshape(-1)])
    gt_rows = np.array(gt, np.float32)
    points = net.points.cpu().numpy()
    ext = synth.extents_for(C)
    sym, flip = np.array([0, 1], np.float32), np.array([0, 1], np.float32)
    ev = Evaluator(C, points, ext, sym, flip_z=flip, device=cuda)
    out = ev.add_poses(T(gt_rows, cuda), dets, {"poses": poses}, None, T(meta, cuda))
    n = int(out["num_pairs"].item())
    d, p = dets.cpu().numpy(), poses.cpu().numpy()
    want = eval_ref.score(gt_rows, d, [p], d.shape[0], meta, points, sym, eval_ref.default_threshold(ext), flip, C)
    np.testing.assert_array_equal(out["pairs"][:n].cpu().numpy(), want[0])
    assert n == int((d[:, 1] == 1).sum()) > 0
    thr = eval_ref.default_threshold(ext)[1]
    amb = check_errors(out["errors"][:, :n].cpu().numpy(), out["flags"][:, :n].cpu().numpy(), want[1], want[2], thr)
    check_counts(ev.counts.cpu().numpy(), want[3], amb)
