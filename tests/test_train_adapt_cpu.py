"""CPU-only checks of the domain-adaptation branch's C ABI entries (pcnn_domain_tail, pcnn_domain_grad_merge): their argument
checks run before any CUDA call, so they are safe without a GPU.  Also the parameter layout of vgg16_convs(adaptation=True)."""
import ctypes

import pytest

MAX_ROWS = 128 * 9


def _tail(lib, buf, rows=9, ld=256, fc9=True, w10=True, b10=True, labels=None, grads=True, outs=True, gscale=1.0):
    p = lambda on: buf if on else None
    return lib.pcnn_domain_tail(p(fc9), rows, ld, p(w10), p(b10), labels, ctypes.c_float(0.1 / max(rows, 1)), ctypes.c_float(gscale),
                                p(outs), p(outs), p(outs), p(grads), p(grads), p(grads), p(grads), p(grads), p(grads), None)


def test_domain_tail_rejects_bad_arguments_without_gpu(native_lib):
    native_lib.pcnn_last_error.restype = ctypes.c_char_p
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    for kw in (dict(fc9=False), dict(w10=False), dict(b10=False), dict(outs=False)):
        assert _tail(native_lib, buf, **kw) == -1, kw
        assert b"NULL" in native_lib.pcnn_last_error()
    assert _tail(native_lib, buf, labels=buf, grads=False) == -1                  # labels without the gradient outputs
    assert b"NULL" in native_lib.pcnn_last_error()
    for rows in (0, -1, MAX_ROWS + 1):
        assert _tail(native_lib, buf, rows=rows) == -1, rows
        assert b"rows" in native_lib.pcnn_last_error()
    for ld in (0, 128, 255, 260, -256):
        assert _tail(native_lib, buf, ld=ld) == -1, ld
        assert b"ld" in native_lib.pcnn_last_error()
    for g in (0.0, -2.0):
        assert _tail(native_lib, buf, labels=buf, gscale=g) == -1, g
        assert b"grad_scale" in native_lib.pcnn_last_error()


def test_domain_grad_merge_rejects_bad_arguments_without_gpu(native_lib):
    native_lib.pcnn_last_error.restype = ctypes.c_char_p
    buf = ctypes.create_string_buffer(64)
    f = ctypes.c_float(1.0)
    for a, b, d in ((None, buf, buf), (buf, None, buf), (buf, buf, None)):
        assert native_lib.pcnn_domain_grad_merge(a, f, b, f, ctypes.c_size_t(8), d, None) == -1
        assert b"NULL" in native_lib.pcnn_last_error()
    for n in (0, 4, 12):
        assert native_lib.pcnn_domain_grad_merge(buf, f, buf, f, ctypes.c_size_t(n), buf, None) == -1, n
        assert b"multiple of 8" in native_lib.pcnn_last_error()


@pytest.mark.parametrize("adaptation,vertex_reg_2d,pose_reg,branch", [(True, True, True, True), (False, True, True, False),
                                                                      (True, True, False, False), (True, False, True, False)])
def test_domain_parameters_follow_fc8(adaptation, vertex_reg_2d, pose_reg, branch):
    """The four parameters exist only where the reference builds the branch, and come after fc8, so the seeded init of every
    other parameter does not move."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(adaptation=adaptation, vertex_reg_2d=vertex_reg_2d, pose_reg=pose_reg, device="cpu")
    assert net.adaptation == adaptation and net.domain_branch == branch
    names = list(net.param_shapes())
    base = list(vgg16_convs(device="cpu").param_shapes())
    extra = ["fc9/weights", "fc9/biases", "domain_score/weights", "domain_score/biases"]
    if branch:
        assert names == base + extra
        shapes = net.param_shapes()
        assert [shapes[k] for k in extra] == [(25088, 256), (256,), (256, 2), (2,)]
    else:
        assert names == base
