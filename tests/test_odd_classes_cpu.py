"""Odd class counts on the CPU (num_classes = 9: the multi-object LINEMOD model, linemod_color_2d.yml): the C ABI's class-count
checks of the up-sampling heads and their adjoint, and the parameter shapes / training layout of vgg16_convs at C = 9 without
pose regression."""
import ctypes

import pytest


def _bwd_ex(native_lib, buf, C, ws_bytes):                     # 2-D target: no vertmap / extents
    f1 = 1.0
    return native_lib.pcnn_up8_heads_bwd(buf, buf, buf, buf, f1, f1, buf, buf, buf, None, None, buf, f1, f1, f1, 1, 60, 80, C, 64, 128,
                                         buf, buf, buf, buf, ws_bytes, None)


def _bwd_coord(native_lib, buf, C, ws_bytes):                  # 3-D target: vertmap and extents given
    f1 = 1.0
    return native_lib.pcnn_up8_heads_bwd(buf, buf, buf, buf, f1, f1, buf, buf, buf, buf, buf, buf, f1, f1, f1, 1, 60, 80, C, 64, 128,
                                         buf, buf, buf, buf, ws_bytes, None)


@pytest.mark.parametrize("entry", [_bwd_ex, _bwd_coord], ids=["2d", "coord"])
def test_up8_backward_accepts_nine_classes(native_lib, entry):
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    # C = 9 passes the class-count check and stops at the workspace check (60 x 80: 20 strips x 4 bands x 36 floats)
    assert entry(native_lib, buf, 9, 16) == -1
    err = native_lib.pcnn_last_error()
    assert b"C must be even" not in err and b"workspace too small (16 < 11520)" in err, err
    for C in (3, 5, 11):                                       # odd counts of no reference configuration: still rejected
        assert entry(native_lib, buf, C, 1 << 20) == -1, C
        assert b"C must be even" in native_lib.pcnn_last_error()


def test_up8_heads_class_range(native_lib):
    buf = ctypes.create_string_buffer(64)
    for C in (1, 129):
        assert native_lib.pcnn_up8_heads(buf, buf, buf, 1, 8, 8, C, buf, buf, None, None, None) == -1, C
        assert b"num_classes must be in 2..128" in native_lib.pcnn_last_error()
    for C in (3, 9, 127):                                      # odd counts pass the class-count check and stop at the shape check (B = 0)
        assert native_lib.pcnn_up8_heads(buf, buf, buf, 0, 8, 8, C, buf, buf, None, None, None) == -1, C
        assert b"up8_heads: bad shape" in native_lib.pcnn_last_error()


def test_nine_class_network_without_pose_reg():
    """linemod_color_2d.yml: NUM_CLASSES 9, VERTEX_REG_2D, POSE_REG False, NUM_UNITS 64."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.train import param_layout
    net = vgg16_convs(num_classes=9, vertex_reg_2d=True, pose_reg=False, device="cpu", is_train=True, fold_vertex_head=False)
    shapes = net.param_shapes()
    assert tuple(shapes["score/weights"]) == (1, 1, 64, 9) and tuple(shapes["score/biases"]) == (9,)
    assert tuple(shapes["vertex_pred/weights"]) == (1, 1, 128, 27) and tuple(shapes["vertex_pred/biases"]) == (27,)
    layout = param_layout(net)
    assert not any(tf.startswith(("fc6", "fc7", "fc8")) for tf, _, _ in layout.values())
    assert {"score/weights", "vertex_pred/weights"} <= {tf for tf, _, _ in layout.values()}
