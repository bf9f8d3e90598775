"""The segmentation network on the CPU: vgg16_convs with vertex_reg_2d and vertex_reg_3d both False has exactly the reference's
variable set, a dictionary of those names loads, the training step's layout trains that set and nothing else, every other
configuration keeps its parameter set, and the new C ABI entries (the score-only heads, pack and adjoint) are declared and check
their arguments before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from posecnn_b200.build import HEADER

# lib/networks/vgg16_convs.py:79-149 (the block at :151-212 is built only under VERTEX_REG_2D / VERTEX_REG_3D): the trainable
# variables of the graph, as (scope, weights shape HWIO, biases shape).  upscore_conv5 / upscore are fixed bilinear filters
# (trainable=False, network.py:207-222), not parameters.
TRUNK = [("conv1_1", (3, 3, 3, 64)), ("conv1_2", (3, 3, 64, 64)),
         ("conv2_1", (3, 3, 64, 128)), ("conv2_2", (3, 3, 128, 128)),
         ("conv3_1", (3, 3, 128, 256)), ("conv3_2", (3, 3, 256, 256)), ("conv3_3", (3, 3, 256, 256)),
         ("conv4_1", (3, 3, 256, 512)), ("conv4_2", (3, 3, 512, 512)), ("conv4_3", (3, 3, 512, 512)),
         ("conv5_1", (3, 3, 512, 512)), ("conv5_2", (3, 3, 512, 512)), ("conv5_3", (3, 3, 512, 512))]


def reference_variables(fmt, C, U=64):
    """{'<scope>/weights' | '<scope>/biases': shape} of the reference's segmentation graph (COLOR: :80-97, 136-149; RGBD adds the
    '_p' trunk of :99-117 and score_conv4 / score_conv5 read the 1024-channel concat, :119-126)."""
    out = {}
    for sfx in ("", "_p") if fmt == "RGBD" else ("",):
        for scope, w in TRUNK:
            out[f"{scope}{sfx}/weights"], out[f"{scope}{sfx}/biases"] = w, (w[3],)
    cin = 1024 if fmt == "RGBD" else 512
    for scope in ("score_conv5", "score_conv4"):
        out[f"{scope}/weights"], out[f"{scope}/biases"] = (1, 1, cin, U), (U,)
    out["score/weights"], out["score/biases"] = (1, 1, U, C), (C,)
    return out


def seg_net(fmt, C, **kw):
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    return vgg16_convs(input_format=fmt, num_classes=C, device="cpu", vertex_reg_2d=False, vertex_reg_3d=False, **kw)


@pytest.mark.parametrize("fmt,C", [("COLOR", 10), ("RGBD", 10), ("COLOR", 8), ("RGBD", 8), ("COLOR", 2), ("COLOR", 22)])
def test_param_shapes_are_the_reference_variables(fmt, C):
    """Also with the constructor's pose_reg / adaptation / fold_vertex_head defaults on or off: the reference ignores them here."""
    for kw in ({}, dict(pose_reg=False), dict(adaptation=True), dict(fold_vertex_head=False), dict(is_train=True)):
        net = seg_net(fmt, C, **kw)
        assert net.param_shapes() == reference_variables(fmt, C), kw
        assert not net.fold_vertex_head and not net.domain_branch


@pytest.mark.parametrize("fmt", ["COLOR", "RGBD"])
def test_train_layout_is_the_reference_variables(fmt):
    from posecnn_b200.train import param_layout, trains_segmentation
    net = seg_net(fmt, 10, is_train=True)
    assert trains_segmentation(net)
    layout = param_layout(net)
    assert sorted(tf for tf, _, _ in layout.values()) == sorted(reference_variables(fmt, 10))
    assert layout["score/w"][2] == 64                     # score's 1x1 GEMM keeps its padded 64 rows


@pytest.mark.parametrize("fmt", ["COLOR", "RGBD"])
def test_reference_dictionary_loads(fmt):
    """A dictionary of exactly the reference's names (flat 'scope/weights' keys, as a TF checkpoint reads) loads and prepares."""
    rng = np.random.default_rng(0)
    d = {k: rng.standard_normal(s).astype(np.float32) for k, s in reference_variables(fmt, 10).items()}
    net = seg_net(fmt, 10).load(d)
    assert set(net.params) == set(d)
    for k, v in d.items():
        assert torch.equal(net.params[k], torch.from_numpy(v)), k
    assert net._tc["score/w"].shape == (64, 10)
    assert "vertex_pred/w" not in net._tc and "fc6/weights" not in net._tc


def _parent_param_shapes(fmt, C, U, domain_branch):
    """The parameter set of every network with a vertex head, restated (it must not change)."""
    out = {}
    for sfx in ("", "_p") if fmt == "RGBD" else ("",):
        for scope, w in TRUNK:
            out[f"{scope}{sfx}/weights"], out[f"{scope}{sfx}/biases"] = w, (w[3],)
    cin = 1024 if fmt == "RGBD" else 512
    for scope, ci, co in (("score_conv5", cin, U), ("score_conv4", cin, U), ("score_conv5_vertex", 512, 128),
                          ("score_conv4_vertex", 512, 128)):
        out[f"{scope}/weights"], out[f"{scope}/biases"] = (1, 1, ci, co), (co,)
    out["score/weights"], out["score/biases"] = (1, 1, U, C), (C,)
    out["vertex_pred/weights"], out["vertex_pred/biases"] = (1, 1, 128, 3 * C), (3 * C,)
    out["fc6/weights"], out["fc6/biases"] = (25088, 4096), (4096,)
    out["fc7/weights"], out["fc7/biases"] = (4096, 4096), (4096,)
    out["fc8/weights"], out["fc8/biases"] = (4096, 4 * C), (4 * C,)
    if domain_branch:
        out["fc9/weights"], out["fc9/biases"] = (25088, 256), (256,)
        out["domain_score/weights"], out["domain_score/biases"] = (256, 2), (2,)
    return out


@pytest.mark.parametrize("fmt", ["COLOR", "RGBD"])
@pytest.mark.parametrize("C", [2, 9, 22])
@pytest.mark.parametrize("v2d,v3d,pose_reg,adapt", [(True, False, True, False), (True, False, False, False), (False, True, True, False),
                                                    (True, True, True, False), (True, False, True, True), (False, True, True, True),
                                                    (False, None, True, False), (False, None, True, True)])
def test_vertex_networks_keep_their_parameters(fmt, C, v2d, v3d, pose_reg, adapt):
    """Also: adaptation builds the domain branch only on a 2-D network with pose_reg (vgg16_convs.py:202-212), and vertex_reg_2d=False
    with vertex_reg_3d left at its default (None) keeps the vertex head: only an explicit vertex_reg_3d=False builds the segmentation
    network."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(input_format=fmt, num_classes=C, device="cpu", vertex_reg_2d=v2d, vertex_reg_3d=v3d, pose_reg=pose_reg,
                      adaptation=adapt)
    shapes = net.param_shapes()
    assert shapes == _parent_param_shapes(fmt, C, 64, net.domain_branch)
    assert list(shapes)[:len(TRUNK) * 2] == [f"{s}/{k}" for s, _ in TRUNK for k in ("weights", "biases")]   # seeded-init order
    assert net.fold_vertex_head == (3 * C <= 128)


NEW_ENTRIES = ("pcnn_lowres_heads_nv", "pcnn_up8_heads_nv", "pcnn_pack_lowres_nv", "pcnn_up8_scores_bwd_workspace_bytes",
               "pcnn_up8_scores_bwd")


def test_header_declares_the_new_entry_points(native_lib):
    from posecnn_b200._lib import prototypes
    with open(HEADER) as f:
        protos = prototypes(f.read())
    for name in NEW_ENTRIES:
        assert name in protos, name
        assert getattr(native_lib, name).argtypes == protos[name][1], name


def test_score_only_entries_reject_bad_arguments_without_gpu(native_lib):
    buf = ctypes.create_string_buffer(1 << 16)                # any non-NULL host address: the checks fail before it is read
    L = native_lib
    # the vertex width is 3C or 0, and the score-only form takes no vertex tensors
    assert L.pcnn_up8_heads_nv(buf, buf, None, 1, 8, 8, 10, 5, buf, None, None, None, None) == -1
    assert b"num_vertex" in L.pcnn_last_error()
    assert L.pcnn_up8_heads_nv(buf, buf, buf, 1, 8, 8, 10, 0, buf, None, None, None, None) == -1
    assert b"no vertex" in L.pcnn_last_error()
    assert L.pcnn_up8_heads_nv(buf, buf, None, 1, 8, 8, 10, 0, buf, buf, None, None, None) == -1
    assert L.pcnn_up8_heads_nv(buf, buf, None, 1, 8, 8, 1, 0, buf, None, None, None, None) == -1
    assert b"num_classes" in L.pcnn_last_error()
    assert L.pcnn_lowres_heads_nv(buf, buf, buf, buf, buf, None, 1, 8, 8, 64, 128, 10, 0, buf, None) == -1
    assert b"no vertex" in L.pcnn_last_error()
    assert L.pcnn_lowres_heads_nv(buf, buf, None, None, buf, None, 1, 8, 8, 64, 0, 10, 29, buf, None) == -1
    assert b"num_vertex" in L.pcnn_last_error()
    assert L.pcnn_lowres_heads_nv(buf, buf, None, None, buf, None, 1, 8, 8, 62, 0, 10, 0, buf, None) == -1
    assert L.pcnn_pack_lowres_nv(buf, 64, buf, 128, 1, 8, 8, 10, 0, buf, None) == -1
    assert L.pcnn_pack_lowres_nv(buf, 8, None, 0, 1, 8, 8, 10, 0, buf, None) == -1
    # the classification-only adjoint: the class counts of pcnn_up8_heads_bwd, a workspace of C floats per CTA
    n = ctypes.c_size_t(0)
    assert L.pcnn_up8_scores_bwd_workspace_bytes(2, 60, 80, 10, ctypes.byref(n)) == 0
    assert n.value == 4 * 2 * 20 * 4 * 10                      # images x strips of 4 cells x bands of 16 rows x C
    m = ctypes.c_size_t(0)
    assert L.pcnn_up8_heads_bwd_workspace_bytes(2, 60, 80, 10, ctypes.byref(m)) == 0 and m.value == 4 * n.value
    assert L.pcnn_up8_scores_bwd_workspace_bytes(1, 60, 80, 2, ctypes.byref(n)) == 0 and n.value == 4 * 5 * 4 * 2   # 16-cell strips
    for C in (1, 3, 4, 7, 11, 52):
        assert L.pcnn_up8_scores_bwd(buf, buf, buf, buf, 1.0, 0.7, 1, 60, 80, C, 64, buf, buf, buf, len(buf), None) == -1, C
        assert b"C must be" in L.pcnn_last_error()
    assert L.pcnn_up8_scores_bwd(buf, buf, buf, buf, 1.0, 0.7, 1, 60, 80, 10, 8, buf, buf, buf, len(buf), None) == -1
    assert b"bad shape" in L.pcnn_last_error()
    assert L.pcnn_up8_scores_bwd(buf, buf, buf, None, 1.0, 0.7, 1, 60, 80, 10, 64, buf, buf, buf, len(buf), None) == -1
    assert b"NULL" in L.pcnn_last_error()
    assert L.pcnn_up8_scores_bwd(buf, buf, buf, buf, 1.0, 0.7, 1, 60, 80, 10, 64, buf, buf, buf, 16, None) == -1
    assert b"workspace too small" in L.pcnn_last_error()
