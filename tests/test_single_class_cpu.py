"""Single-object (num_classes = 2) models on the CPU: the up-sampling adjoint's C ABI accepts C = 2, the pose_reg=False layout
table holds exactly the reference's variables, and the two-class data view and its inverse equal the reference's own lines
(tests/golden/single_class.npz, made by tests/golden/make_golden_single_class.py)."""
import ctypes
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "single_class.npz")


def test_up8_backward_accepts_two_classes(native_lib):
    f1 = 1.0
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    # C = 2 passes the class-count check and stops at the workspace check (the 60 x 80 problem needs 5 x 4 CTAs x 8 floats)
    assert native_lib.pcnn_up8_heads_bwd_ex(buf, buf, buf, buf, f1, f1, buf, None, None, buf, buf, f1, f1, f1, 1, 60, 80, 2, 64, 128,
                                            buf, buf, buf, buf, 16, None) == -1
    err = native_lib.pcnn_last_error()
    assert b"C must be even" not in err and b"workspace too small (16 < 640)" in err, err
    for C in (4, 7, 23, 52):                                   # no reference configuration uses them: still rejected
        assert native_lib.pcnn_up8_heads_bwd_ex(buf, buf, buf, buf, f1, f1, buf, None, None, buf, buf, f1, f1, f1, 1, 8, 8, C, 64, 160,
                                                buf, buf, buf, buf, 1 << 20, None) == -1, C
        assert b"C must be even" in native_lib.pcnn_last_error()


def test_pose_reg_false_layout_is_the_reference_variables():
    """vgg16_convs.py:79-163 creates these variables; fc6-fc8 exist only under POSE_REG (vgg16_convs.py:175-200)."""
    from posecnn_b200.networks.vgg16_convs import VGG_CFG, vgg16_convs
    from posecnn_b200.train import param_layout
    trunk = [item[0] for item in VGG_CFG if isinstance(item, tuple)]
    heads = ["score_conv5", "score_conv4", "score_conv5_vertex", "score_conv4_vertex", "score", "vertex_pred"]
    want = sorted(f"{layer}/{kind}" for layer in trunk + heads for kind in ("weights", "biases"))
    for C, adaptation in ((2, False), (2, True), (22, False)):
        net = vgg16_convs(num_classes=C, device="cpu", is_train=True, fold_vertex_head=False, pose_reg=False, adaptation=adaptation)
        layout = param_layout(net)
        assert sorted(tf for tf, _, _ in layout.values()) == want
        assert sorted(layout) == sorted(f"{n}/{k}" for n in trunk + heads for k in ("w", "b"))
        assert {"fc6/weights", "fc7/weights", "fc8/weights"} <= set(net.param_shapes())     # the seeded init is unchanged
    net = vgg16_convs(num_classes=2, device="cpu", is_train=True, fold_vertex_head=False)
    assert sorted(tf for tf, _, _ in param_layout(net).values()) == sorted(net.param_shapes())


def _quat_cols(poses, k):
    return poses[0, :, k]                                      # any four values that travel with the row


def test_single_class_view_equals_reference_lines():
    from posecnn_b200.single_class import single_class_view
    g = np.load(GOLDEN)
    cls, C, B = int(g["cls_index"]), int(g["num_classes_all"]), int(g["batch"])
    H, W = g["in0_label"].shape
    label = np.stack([g[f"in{b}_label"].astype(np.int32) for b in range(B)])
    label[1, 0, :5] = -1                                       # ignored pixels stay ignored
    centers = np.zeros((B, C, 3), np.float32)
    rows = []
    for b in range(B):
        poses = g[f"in{b}_poses"]
        for k, c in enumerate(g[f"in{b}_cls_indexes"].flatten().astype(int)):
            centers[b, c] = (*g[f"in{b}_center"][k], poses[2, 3, k])
            rows.append([b, c, *g[f"in{b}_box"][k], *_quat_cols(poses, k), *poses[:, 3, k]])
    gt = np.asarray(rows, np.float32)
    rng = np.random.default_rng(3)
    ext, pts, sym = rng.random((C, 3)).astype(np.float32), rng.random((C, 50, 3)).astype(np.float32), (np.arange(C) % 3 == 0).astype(np.float32)
    T = torch.from_numpy
    v = single_class_view(cls, T(label), T(centers), T(gt), T(ext), T(pts), T(sym))
    want_label = np.stack([g[f"out{b}_label"].astype(np.int32) for b in range(B)])
    want_label[1, 0, :5] = -1
    assert v["label"].dtype == torch.int32 and np.array_equal(v["label"].numpy(), want_label)
    want_rows, want_centers = [], np.zeros((B, 2, 3), np.float32)
    for b in range(B):
        poses, ind = g[f"out{b}_poses"], g[f"out{b}_ind"]
        assert np.array_equal(g[f"out{b}_poses"], g[f"in{b}_poses"][:, :, ind])
        for k in range(len(ind)):
            want_rows.append([b, g[f"out{b}_cls_indexes"][k], *g[f"out{b}_box"][k], *_quat_cols(poses, k), *poses[:, 3, k]])
            want_centers[b, 1] = (*g[f"out{b}_center"][k], poses[2, 3, k])
    assert len(want_rows) == 3                                 # image 2 does not show the object
    assert np.array_equal(v["gt_poses"].numpy(), np.asarray(want_rows, np.float32))
    assert np.array_equal(v["centers"].numpy(), want_centers)
    # the two-row tables of lib/datasets/linemod.py:30-51,167-195 (extents with the background row, lov.py:168)
    assert np.array_equal(v["extents"].numpy(), np.stack([np.zeros(3, np.float32), ext[cls]]))
    assert np.array_equal(v["points"].numpy(), np.stack([np.zeros((50, 3), np.float32), pts[cls]]))
    assert np.array_equal(v["symmetry"].numpy(), np.array([0.0, sym[cls]], np.float32))
    assert np.array_equal(label[0], np.stack([g[f"in{b}_label"] for b in range(B)])[0])    # the inputs are not changed


def test_inverse_equals_reference_lines():
    from posecnn_b200.utils.results import to_dataset_classes
    g = np.load(GOLDEN)
    cls = int(g["cls_index"])
    rois_in = g["icp_rois_in"].copy()
    for b in range(int(g["batch"])):
        lab_in = g["icp_labels_in"][b].copy()
        labels, rois = to_dataset_classes(lab_in, rois_in, cls)
        assert np.array_equal(labels, g["icp_labels_out"][b]) and labels.dtype == np.int32
        assert np.array_equal(rois, g["icp_rois_out"])
        assert np.array_equal(lab_in, g["icp_labels_in"][b]) and np.array_equal(rois_in, g["icp_rois_in"])
