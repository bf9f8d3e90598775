// TEST INFRASTRUCTURE ONLY.  The reference's GPU NMS (lib/nms/nms_kernel.cu, the kernel behind gpu_nms.pyx that
// lib/rpn_layer/proposal_layer.py runs with cfg.USE_GPU_NMS = True), #included unmodified from the reference checkout and
// compiled with nvcc's defaults as the reference's setup.py compiles it (FMA contraction on).  Built by ref_nms.mk into
// _ref/libref_nms.so; tests/test_det_gpu.py compares the device's proposal NMS against it.
#define REF_STR2(x) #x
#define REF_STR(x) REF_STR2(x)
#include REF_STR(REF_ROOT/lib/nms/nms_kernel.cu)

// boxes_host [n,5] f32 (x1, y1, x2, y2, score) already in processing order (gpu_nms.pyx sorts before calling _nms);
// keep_out [n] receives the kept row indices in order, *num_out their count.  Synchronous, on the default stream.
extern "C" int ref_gpu_nms(int* keep_out, int* num_out, const float* boxes_host, int n, float thresh, int device_id)
{
    if (!keep_out || !num_out || !boxes_host || n < 1) return -1;
    _nms(keep_out, num_out, boxes_host, n, 5, thresh, device_id);
    return cudaGetLastError() == cudaSuccess ? 0 : -3;
}
