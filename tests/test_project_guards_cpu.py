"""CPU-only checks of the 32-bit index guards of Backproject / Project and their gradients (csrc/pixel_ops.cu launch_gather and
launch_average): the kernels index inside one image with 32-bit unsigned arithmetic and put the image on grid.y, so a grid or
image of 2^31 - 1 or more elements per image, or more than 65535 images, is rejected before any CUDA call.  Every shape here
is rejected before a launch, so host buffers stand in for the tensors and no GPU is needed."""
import ctypes

import pytest

PCNN_OK, PCNN_E_INVALID = 0, -1


@pytest.fixture
def buf():
    """A small host buffer: non-NULL for the pointer checks, never read, and filled with a sentinel so that a call which
    returns early can be seen to have written nothing."""
    b = (ctypes.c_float * 64)(*([7.0] * 64))
    return ctypes.cast(b, ctypes.POINTER(ctypes.c_float)), b


def _rejected(lib, rc, what):
    assert rc == PCNN_E_INVALID, rc
    assert what in lib.pcnn_last_error(), lib.pcnn_last_error()


def test_backproject_fwd_grid_of_2_31_elements(native_lib, buf):
    """G = 512, Cf = 16 (the GRID_SIZE of the 512-grid reference configurations): G^3 * Cf = 2^31.  The fused kernel is
    skipped (G^3 * max(Cf, C) >= 2^31 - 1) and the data pass's guard rejects; C = 3 alone would pass."""
    p, _ = buf
    for Cf in (16, 17, 64):
        rc = native_lib.pcnn_backproject_fwd(p, p, p, p, p, 1, 8, 8, Cf, 3, 48, 512, 3, 0.02, p, p, p, None)
        _rejected(native_lib, rc, b"32-bit indexing")


def test_project_bwd_grid_of_2_31_elements(native_lib, buf):
    p, _ = buf
    rc = native_lib.pcnn_project_bwd(p, p, p, 1, 8, 8, 16, 48, 512, 3, 0.02, p, None)
    _rejected(native_lib, rc, b"32-bit indexing")


@pytest.mark.parametrize("H,W,Cf", [(8192, 4096, 64), (32768, 32768, 2), (46341, 46341, 1)])
def test_gathers_with_2_31_elements_per_image(native_lib, buf, H, W, Cf):
    """Project forward and BackprojectGrad (one pixel gather) with H * W * Cf >= 2^31 - 1."""
    p, _ = buf
    assert H * W * Cf >= 0x7fffffff
    _rejected(native_lib, native_lib.pcnn_project_fwd(p, p, p, 1, H, W, Cf, 48, 16, p, None), b"32-bit indexing")
    _rejected(native_lib, native_lib.pcnn_backproject_bwd(p, p, p, 1, H, W, Cf, 48, 16, p, None), b"32-bit indexing")


def test_batch_of_65536_images(native_lib, buf):
    """grid.y holds the image: B = 65536 is rejected by all four entries (Backproject through its data pass: the fused
    kernel is skipped for B > 65535)."""
    p, _ = buf
    B = 65536
    _rejected(native_lib, native_lib.pcnn_backproject_fwd(p, p, p, p, p, B, 8, 8, 4, 3, 48, 4, 1, 0.02, p, p, p, None),
              b"32-bit indexing")
    _rejected(native_lib, native_lib.pcnn_project_bwd(p, p, p, B, 8, 8, 4, 48, 4, 1, 0.02, p, None), b"32-bit indexing")
    _rejected(native_lib, native_lib.pcnn_project_fwd(p, p, p, B, 8, 8, 4, 48, 4, p, None), b"32-bit indexing")
    _rejected(native_lib, native_lib.pcnn_backproject_bwd(p, p, p, B, 8, 8, 4, 48, 4, p, None), b"32-bit indexing")


def test_backproject_fwd_grid_size_zero_does_nothing(native_lib, buf):
    """grid_size 0 is a valid argument of the reference op (backprojecting_op.cc:303-305) and gives empty outputs: PCNN_OK,
    nothing written, no launch."""
    p, raw = buf
    assert native_lib.pcnn_backproject_fwd(p, p, p, p, p, 2, 8, 8, 4, 3, 48, 0, 3, 0.02, p, p, p, None) == PCNN_OK
    assert list(raw) == [7.0] * 64
