"""CPU-only checks of the RGB-D training step's new C ABI entry (pcnn_im2col_depth): its argument checks run before any CUDA
call, so they are safe without a GPU."""
import ctypes


def test_im2col_depth_rejects_bad_arguments_without_gpu(native_lib):
    native_lib.pcnn_last_error.restype = ctypes.c_char_p
    mean = (ctypes.c_float * 3)(102.9801, 115.9465, 122.7717)
    buf = ctypes.create_string_buffer(64)                      # any non-NULL host address: the checks fail before it is read
    assert native_lib.pcnn_im2col_depth(None, mean, buf, 1, 8, 8, None) == -1
    assert b"NULL" in native_lib.pcnn_last_error()
    assert native_lib.pcnn_im2col_depth(buf, mean, None, 1, 8, 8, None) == -1
    assert b"NULL" in native_lib.pcnn_last_error()
    for B, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, 0), (-1, 8, 8), (1, 8, -4)):
        assert native_lib.pcnn_im2col_depth(buf, mean, buf, B, H, W, None) == -1, (B, H, W)
        assert b"bad shape" in native_lib.pcnn_last_error()
    assert native_lib.pcnn_im2col_depth(buf, mean, buf, 1, 65536, 8, None) == -1
    assert b"too tall" in native_lib.pcnn_last_error()
    assert native_lib.pcnn_im2col_depth(buf, mean, buf, 65536, 8, 8, None) == -1
