"""Object-coordinate (VERTEX_REG_3D) training on the CPU: the numpy restatement of the 3-D target equals the reference's own
_generate_vertex_targets / _scale_vertmap bit for bit (tests/golden/vertex_targets_3d.npz, made by
tests/golden/make_golden_vertex_3d.py), the new C entry points check their arguments like their 2-D twins, and the parameter
layout of the 3-D graph has no pose head."""
import ctypes
import os

import numpy as np

from tests.train_coord_ref import presence_table, vertex_targets_3d

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vertex_targets_3d.npz")


def load_golden():
    g = np.load(GOLDEN)
    cen = presence_table([g["cls_indexes0"], g["cls_indexes1"]], g["extents"].shape[0])
    return g, cen


def test_restatement_equals_reference_golden():
    g, cen = load_golden()
    t, w = vertex_targets_3d(g["label"], g["vertmap"], cen, g["extents"], float(g["w_inside"]))
    assert np.array_equal(t.view(np.int32), g["targets"].view(np.int32))
    assert np.array_equal(w, g["weights"])
    # the cases the vectors cover: an unlisted class with pixels, a listed class without, a zero and a negative extent axis
    lab, wt = g["label"], g["weights"]
    assert (lab[0] == 3).any() and not wt[0, ..., 9:12].any()
    assert not (lab[0] == 4).any() and cen[0, 4, 2] > 0
    assert (lab[0] == 2).any() and wt[0, ..., 7].any() and not g["targets"][0, ..., 7].any()
    assert (lab[1] == 5).any() and wt[1, ..., 17].any() and not g["targets"][1, ..., 17].any()
    assert len({int(c) for c in np.unique(lab[1]) if c > 0}) >= 3


def test_coord_target_and_loss_entries_check_arguments(native_lib):
    f1 = 1.0
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    ws = 1 << 20
    # targets: every tensor is required; shapes positive
    assert native_lib.pcnn_vertex_targets_3d_fwd(buf, None, buf, buf, 1, 8, 8, 6, f1, buf, buf, None) == -1
    assert b"vertex_targets_3d: NULL tensor pointer" in native_lib.pcnn_last_error()
    assert native_lib.pcnn_vertex_targets_3d_fwd(buf, buf, buf, buf, 1, 0, 8, 6, f1, buf, buf, None) == -1
    assert b"vertex_targets_3d: bad shape" in native_lib.pcnn_last_error()
    assert native_lib.pcnn_vertex_targets_3d_fwd(buf, buf, buf, buf, 65536, 256, 256, 6, f1, buf, buf, None) == -1
    assert b"too many pixels" in native_lib.pcnn_last_error()
    # fused loss: the head tensor and its bias are required; vertmap and extents go together; sigma > 0; H, W % 8 == 0; workspace size
    def loss(lowres, bias, vertmap, extents, H=64, sigma=f1, ws=ws):
        return native_lib.pcnn_vertex_loss_fwd(lowres, bias, buf, buf, vertmap, extents, 1, H, 96, 22, f1, sigma, buf, buf, ws, None)
    assert loss(buf, None, buf, buf) == -1 and b"vertex_loss: NULL tensor pointer" in native_lib.pcnn_last_error()
    assert loss(None, buf, buf, buf) == -1 and b"vertex_loss: NULL tensor pointer" in native_lib.pcnn_last_error()
    assert loss(buf, buf, None, buf) == -1 and b"vertex_loss: vertmap and extents" in native_lib.pcnn_last_error()
    assert loss(buf, buf, buf, None) == -1 and b"vertex_loss: vertmap and extents" in native_lib.pcnn_last_error()
    assert loss(buf, buf, buf, buf, sigma=0.0) == -1 and b"vertex_loss: bad arguments" in native_lib.pcnn_last_error()
    assert loss(buf, buf, buf, buf, ws=16) == -1 and b"vertex_loss: workspace too small" in native_lib.pcnn_last_error()
    assert loss(buf, buf, buf, buf, H=60) == -1 and b"vertex_loss: bad arguments" in native_lib.pcnn_last_error()
    assert loss(buf, buf, None, None, H=60) == -1 and b"vertex_loss: bad arguments" in native_lib.pcnn_last_error()   # 2-D target


def test_coord_adjoint_checks_arguments(native_lib):
    f1 = 1.0
    buf = ctypes.create_string_buffer(64)

    def call(vertmap, extents, C, h=8, w=8, ws=1 << 20, lowres=buf):
        return native_lib.pcnn_up8_heads_bwd(buf, buf, buf, buf, f1, f1, lowres, buf, buf, vertmap, extents, buf, f1, f1, f1, 1, h, w, C, 64,
                                             160, buf, buf, buf, buf, ws, None)
    assert call(None, buf, 22) == -1 and b"up8_heads_bwd: vertmap and extents" in native_lib.pcnn_last_error()
    assert call(buf, None, 22) == -1 and b"up8_heads_bwd: vertmap and extents" in native_lib.pcnn_last_error()
    for vm in (None, buf):                                     # the low-resolution head tensor is required in both target modes
        assert call(vm, vm, 22, lowres=None) == -1 and b"up8_heads_bwd: NULL tensor pointer" in native_lib.pcnn_last_error()
    for C in (4, 7, 23, 52):                                   # the class counts of the 2-D target, no others
        assert call(buf, buf, C) == -1, C
        assert b"C must be even" in native_lib.pcnn_last_error()
    # C = 2 (16-cell strips: 5 x 4 CTAs x 8 floats at 60 x 80) passes the class-count check and stops at the workspace check
    assert call(buf, buf, 2, 60, 80, 16) == -1
    err = native_lib.pcnn_last_error()
    assert b"C must be even" not in err and b"workspace too small (16 < 640)" in err, err


def test_coord_layout_has_no_pose_head():
    """The reference builds Hough voting, RoiPool and fc6-fc8 only under vertex_reg_2d (vgg16_convs.py:165-200): an object-coordinate
    network trains the trunk and the dense heads alone, whatever pose_reg says."""
    from posecnn_b200.networks.vgg16_convs import VGG_CFG, vgg16_convs
    from posecnn_b200.train import param_layout, trains_coords
    trunk = [item[0] for item in VGG_CFG if isinstance(item, tuple)]
    heads = ["score_conv5", "score_conv4", "score_conv5_vertex", "score_conv4_vertex", "score", "vertex_pred"]
    want = sorted(f"{layer}/{kind}" for layer in trunk + heads for kind in ("weights", "biases"))
    for C in (2, 22):
        for pose_reg in (True, False):
            net = vgg16_convs(num_classes=C, device="cpu", is_train=True, fold_vertex_head=False, vertex_reg_2d=False, vertex_reg_3d=True,
                              pose_reg=pose_reg)
            assert trains_coords(net)
            assert sorted(tf for tf, _, _ in param_layout(net).values()) == want
    net = vgg16_convs(num_classes=22, device="cpu", is_train=True, fold_vertex_head=False, vertex_reg_2d=True, vertex_reg_3d=True)
    assert not trains_coords(net) and "fc8/w" in param_layout(net)    # a 2-D network trains as before
