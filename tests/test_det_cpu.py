"""CPU-only checks of the detection network (vgg16_det): anchors and the proposal-layer restatement against tests/golden/det.npz
(the reference's own rpn_layer code, tests/golden/make_golden_det.py), the parameter table, and the argument checks of the
new native entry points, which reject bad input before any CUDA work."""
import ctypes
import os

import numpy as np
import pytest

from posecnn_b200.rpn_layer.snippets import generate_anchors_pre
from tests import det_ref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "det.npz"))
CASES = {"lov": (30, 40, (4, 8, 16, 32)), "linemod": (30, 40, (3, 4, 5, 6, 7, 8)), "small": (5, 7, (4, 8, 16, 32)),
         "few": (4, 5, (4, 8, 16, 32))}
RATIOS = (0.5, 0.75, 1, 1.5, 2)


def golden_inputs(tag):
    """rpn_cls_prob [h,w,2A] and rpn_bbox_pred [h,w,4A] f32 of a golden case."""
    fg = GOLD[f"{tag}_fg"][0]
    return np.concatenate([np.float32(1) - fg, fg], axis=-1), GOLD[f"{tag}_deltas"][0].astype(np.float32)


@pytest.mark.parametrize("tag", sorted(CASES))
def test_anchors_equal_reference(tag):
    h, w, scales = CASES[tag]
    anchors, n = generate_anchors_pre(h, w, 16, scales, RATIOS)
    assert anchors.dtype == np.float32 and int(n) == h * w * len(scales) * len(RATIOS)
    np.testing.assert_array_equal(anchors, GOLD[f"{tag}_anchors"])


@pytest.mark.parametrize("tag", sorted(CASES))
def test_proposal_restatement_equals_reference(tag):
    prob, deltas = golden_inputs(tag)
    im_h, im_w = GOLD[f"{tag}_im"]
    rois, scores, _, _ = det_ref.proposal_layer(prob, deltas, GOLD[f"{tag}_anchors"], im_h, im_w)
    g_rois, g_scores = GOLD[f"{tag}_rois"], GOLD[f"{tag}_scores"]
    assert (g_rois[:, 0] == 0).all()
    np.testing.assert_array_equal(rois, g_rois[:, 1:])
    np.testing.assert_array_equal(scores, g_scores[:, 0])


def test_golden_cases_cover_the_limits():
    assert GOLD["lov_rois"].shape[0] == 300 and GOLD["linemod_rois"].shape[0] == 300
    assert GOLD["small_anchors"].shape[0] < 6000 and GOLD["few_rois"].shape[0] < 300


def test_canonical_order_breaks_ties_by_index():
    s = np.array([0.5, 0.7, 0.5, 0.5, 0.9], dtype=np.float32)
    assert det_ref.canonical_order(s).tolist() == [4, 1, 0, 2, 3]


@pytest.mark.parametrize("C,scales", [(22, (4, 8, 16, 32)), (2, (3, 4, 5, 6, 7, 8))])
def test_param_shapes_follow_reference(C, scales):
    from posecnn_b200.networks import vgg16_det
    net = vgg16_det(num_classes=C, anchor_scales=scales, device="cpu")
    A = len(scales) * 5
    s = net.param_shapes()
    assert net.num_anchors == A
    assert s["conv1_1/weights"] == (3, 3, 3, 64) and s["conv5_3/weights"] == (3, 3, 512, 512)
    assert s["conv_rpn/weights"] == (3, 3, 512, 512)
    assert s["rpn_cls_score/weights"] == (1, 1, 512, 2 * A) and s["rpn_bbox_pred/weights"] == (1, 1, 512, 4 * A)
    assert s["fc6/weights"] == (25088, 4096) and s["fc7/weights"] == (4096, 4096)
    assert s["cls_score/weights"] == (4096, C) and s["bbox_pred/weights"] == (4096, 4 * C)
    assert s["poses_pred_unnormalized/weights"] == (4096, 4 * C)
    layers = {k.split("/")[0] for k in s}
    assert len(layers) == 13 + 8 and all(f"{n}/biases" in s for n in layers)


def test_non_colour_input_is_rejected():
    from posecnn_b200.networks import vgg16_det
    with pytest.raises(ValueError):
        vgg16_det(input_format="RGBD", device="cpu")


def test_entry_points_reject_bad_arguments(native_lib):
    buf = ctypes.create_string_buffer(256)
    nbytes = ctypes.c_size_t(0)
    err = lambda: native_lib.pcnn_last_error()
    assert native_lib.pcnn_rpn_heads_fwd(buf, buf, buf, 10, 65, buf, buf, None) == -1 and b"A = 65" in err()
    assert native_lib.pcnn_rpn_heads_fwd(buf, buf, buf, 0, 20, buf, buf, None) == -1 and b"non-positive" in err()
    assert native_lib.pcnn_rpn_proposals_workspace_bytes(1, 30, 40, 65, 6000, ctypes.byref(nbytes)) == -1 and b"A = 65" in err()
    assert native_lib.pcnn_rpn_proposals_workspace_bytes(0, 30, 40, 20, 6000, ctypes.byref(nbytes)) == -1
    assert native_lib.pcnn_rpn_proposals_workspace_bytes(1, 30, 0, 20, 6000, ctypes.byref(nbytes)) == -1
    assert native_lib.pcnn_rpn_proposals_workspace_bytes(1, 30, 40, 20, 0, ctypes.byref(nbytes)) == -1 and b"pre_top_n" in err()
    assert native_lib.pcnn_rpn_proposals_workspace_bytes(1, 30, 40, 20, 16385, ctypes.byref(nbytes)) == -1
    # pre_top_n is clamped to the anchor count, as the reference's slice: 7 x 5 x 20 = 700 candidates, 11 mask words each
    assert native_lib.pcnn_rpn_proposals_workspace_bytes(1, 5, 7, 20, 6000, ctypes.byref(nbytes)) == 0
    K = 700
    assert nbytes.value >= K * 16 + K * 4 + K * 11 * 8 and nbytes.value < 6000 * 16
    args = lambda B, A, post, ws: (buf, buf, buf, B, 30, 40, A, 480.0, 640.0, 6000, post, 0.7, buf, buf, buf, None, buf, ws, None)
    assert native_lib.pcnn_rpn_proposals_fwd(*args(1, 65, 300, 1 << 30)) == -1 and b"A = 65" in err()
    assert native_lib.pcnn_rpn_proposals_fwd(*args(0, 20, 300, 1 << 30)) == -1
    assert native_lib.pcnn_rpn_proposals_fwd(*args(1, 20, 0, 1 << 30)) == -1 and b"post_top_n" in err()
    assert native_lib.pcnn_rpn_proposals_fwd(*args(1, 20, 300, 16)) == -2 and b"workspace too small" in err()
    assert native_lib.pcnn_crop_pool_f16(buf, 1, 30, 40, 12, buf, 10, 5, 16.0, buf, None) == -1 and b"C = 12" in err()
    assert native_lib.pcnn_crop_pool_f16(buf, 1, 30, 40, 512, buf, 0, 5, 16.0, buf, None) == -1
    assert native_lib.pcnn_crop_pool_f16(buf, 1, 30, 40, 512, buf, 10, 4, 16.0, buf, None) == -1
    assert native_lib.pcnn_softmax_rows_f32(buf, 0, 22, buf, None) == -1
