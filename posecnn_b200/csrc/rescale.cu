// rescale.cu — the image-scale resizes of SCALES_BASE != 1 on the device: cv2.resize(x, None, None, fx=s, fy=s, interpolation)
// as the reference applies it at test time (lib/fcn/test.py:49-65 colour blob, :1335 / :1384 raw depth, :1421 labels back to the
// frame) and in training (lib/gt_synthesize_layer/minibatch.py:179-183 colour blob, :352 label image, :416 vertmap).
//
// The arithmetic is OpenCV's generic (non-SIMD) resize, bit for bit (tests/rescale_ref.py restates it):
//   LINEAR   f = float((d + 0.5) * (1 / fx) - 0.5) in double, s = floor(f), a = f - s (float).  Columns: s < 0 -> (0, a = 0),
//            s >= W - 1 -> (W - 1, a = 0), second tap min(s + 1, W - 1).  Rows: only the indices s, s + 1 are clamped to
//            [0, H - 1]; the row weight is never zeroed.  h = RN(RN(S0 (1 - a)) + RN(S1 a)) per source row, then
//            out = RN(RN(h0 (1 - b)) + RN(h1 b)), float32 with no FMA (every step spelled with the _rn intrinsics).
//            uint16 output (depth): round half to even, saturate to [0, 65535].
//   NEAREST  s = min(floor(d * (1 / fx)), n - 1) in double.
// One CTA per output row of one image; the threads stride over the row's W_out * C elements, so stores are coalesced.  Offsets
// of rows and images are 64-bit; indices inside a row are int, so a row of W * C or W_out * C elements above INT_MAX is refused.
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace pcnn {
namespace rescale {

constexpr int kThreads = 256;

struct Mean3 {
    double m0, m1, m2;
};

// cv2's source coordinate of destination index d: f = float((d + 0.5) * scale - 0.5), s = floor(f), a = f - s
__device__ __forceinline__ void lin_coord(int d, double scale, int& s, float& a)
{
    const float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
    s = (int)floorf(f);
    a = __fsub_rn(f, (float)s);
}

// source value as the float32 the reference resizes: f32(f64(u8) - mean) (the augment.cu convention), f32, or f32(u16)
__device__ __forceinline__ float src_value(const uint8_t* p, size_t i, int c, const Mean3& m)
{
    return __double2float_rn(__dsub_rn((double)p[i], c == 0 ? m.m0 : (c == 1 ? m.m1 : m.m2)));
}
__device__ __forceinline__ float src_value(const float* p, size_t i, int, const Mean3&) { return p[i]; }
__device__ __forceinline__ float src_value(const uint16_t* p, size_t i, int, const Mean3&) { return (float)p[i]; }

// saturate_cast<ushort>(float): cvRound (half to even), then clamp; NaN rounds to INT_MIN and saturates to 0
__device__ __forceinline__ int round_u16(float v) { return min(max(__float2int_rn(v), 0), 65535); }

__device__ __forceinline__ void store(float* p, size_t i, float v, bool round_depth)
{
    p[i] = round_depth ? (float)round_u16(v) : v;
}
__device__ __forceinline__ void store(uint16_t* p, size_t i, float v, bool) { p[i] = (uint16_t)round_u16(v); }

template <int C, typename Src, typename Dst>
__global__ void __launch_bounds__(kThreads)
k_resize_linear(const Src* __restrict__ src, int H, int W, double scale, int Wo, Mean3 mean, bool round_depth, Dst* __restrict__ dst)
{
    const int dy = blockIdx.x, b = blockIdx.y, Ho = gridDim.x;
    int sy;
    float fb;
    lin_coord(dy, scale, sy, fb);
    const int y0 = min(max(sy, 0), H - 1), y1 = min(max(sy + 1, 0), H - 1);
    const float b0 = __fsub_rn(1.f, fb);
    const size_t row = (size_t)W * C;
    const Src* r0 = src + ((size_t)b * H + y0) * row;
    const Src* r1 = src + ((size_t)b * H + y1) * row;
    const size_t out = ((size_t)b * Ho + dy) * ((size_t)Wo * C);
    for (int e = threadIdx.x; e < Wo * C; e += kThreads) {
        const int dx = e / C, c = e - dx * C;
        int sx;
        float fa;
        lin_coord(dx, scale, sx, fa);
        if (sx < 0) { sx = 0; fa = 0.f; }
        if (sx >= W - 1) { sx = W - 1; fa = 0.f; }
        const int i0 = sx * C + c, i1 = min(sx + 1, W - 1) * C + c;
        const float a0 = __fsub_rn(1.f, fa);
        const float h0 = __fadd_rn(__fmul_rn(src_value(r0, i0, c, mean), a0), __fmul_rn(src_value(r0, i1, c, mean), fa));
        const float h1 = __fadd_rn(__fmul_rn(src_value(r1, i0, c, mean), a0), __fmul_rn(src_value(r1, i1, c, mean), fa));
        store(dst, out + e, __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, fb)), round_depth);
    }
}

__global__ void __launch_bounds__(kThreads)
k_resize_nearest(const int32_t* __restrict__ src, int H, int W, double inv, int Wo, int32_t* __restrict__ dst)
{
    const int dy = blockIdx.x, b = blockIdx.y, Ho = gridDim.x;
    const int sy = min((int)floor(__dmul_rn((double)dy, inv)), H - 1);
    const int32_t* r = src + ((size_t)b * H + sy) * W;
    int32_t* o = dst + ((size_t)b * Ho + dy) * Wo;
    for (int dx = threadIdx.x; dx < Wo; dx += kThreads) o[dx] = r[min((int)floor(__dmul_rn((double)dx, inv)), W - 1)];
}

}  // namespace rescale
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::rescale;

// The destination must be cv2's: round(H * fx) x round(W * fx) with round half to even (saturate_cast<int>(double)).
static int check_resize(const char* what, int B, int H, int W, int C, double fx, int Ho, int Wo)
{
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "%s: bad shape B=%d H=%d W=%d", what, B, H, W);
    PCNN_REQUIRE(B <= 65535, "%s: B must be <= 65535 (got %d)", what, B);
    PCNN_REQUIRE(isfinite(fx) && fx > 0.0, "%s: fx must be finite and > 0 (got %g)", what, fx);
    const double hs = (double)H * fx, ws = (double)W * fx;
    PCNN_REQUIRE(hs < (double)INT_MAX && ws < (double)INT_MAX, "%s: %d x %d scaled by %g is too large", what, H, W, fx);
    const long long ho = llrint(hs), wo = llrint(ws);
    PCNN_REQUIRE(ho >= 1 && wo >= 1, "%s: %d x %d scaled by %g is empty", what, H, W, fx);
    PCNN_REQUIRE(Ho == ho && Wo == wo, "%s: destination must be round(H * fx) x round(W * fx) = %lld x %lld (got %d x %d)", what, ho,
                 wo, Ho, Wo);
    PCNN_REQUIRE((long long)W * C <= INT_MAX && (long long)Wo * C <= INT_MAX,
                 "%s: a row of %d (source) or %d (destination) x %d channels overflows the kernel's int row index", what, W, Wo, C);
    return PCNN_OK;
}

template <int C, typename Src, typename Dst>
static int launch_linear(const Src* src, int B, int H, int W, double fx, int Ho, int Wo, Mean3 mean, bool round_depth, Dst* dst,
                         void* stream, const char* what)
{
    k_resize_linear<C, Src, Dst><<<dim3(Ho, B), kThreads, 0, (cudaStream_t)stream>>>(src, H, W, 1.0 / fx, Wo, mean, round_depth, dst);
    return check_launch(what);
}

extern "C" int pcnn_resize_color_u8(const uint8_t* frames, int B, int H, int W, double fx, int Ho, int Wo, const double* mean3_host,
                                    float* blob, void* stream)
{
    PCNN_REQUIRE(frames && blob && mean3_host, "resize_color_u8: NULL tensor pointer");
    if (int rc = check_resize("resize_color_u8", B, H, W, 3, fx, Ho, Wo)) return rc;
    const Mean3 m{mean3_host[0], mean3_host[1], mean3_host[2]};
    return launch_linear<3>(frames, B, H, W, fx, Ho, Wo, m, false, blob, stream, "resize_color_u8");
}

extern "C" int pcnn_resize_linear_f32(const float* src, int B, int H, int W, int C, double fx, int Ho, int Wo, float* dst, void* stream)
{
    PCNN_REQUIRE(src && dst, "resize_linear_f32: NULL tensor pointer");
    PCNN_REQUIRE(C == 1 || C == 3, "resize_linear_f32: C must be 1 or 3 (got %d)", C);
    if (int rc = check_resize("resize_linear_f32", B, H, W, C, fx, Ho, Wo)) return rc;
    const Mean3 m{0.0, 0.0, 0.0};
    return C == 1 ? launch_linear<1>(src, B, H, W, fx, Ho, Wo, m, false, dst, stream, "resize_linear_f32")
                  : launch_linear<3>(src, B, H, W, fx, Ho, Wo, m, false, dst, stream, "resize_linear_f32");
}

extern "C" int pcnn_resize_depth(const void* depth, int depth_is_u16, int B, int H, int W, double fx, int Ho, int Wo, void* dst,
                                 void* stream)
{
    PCNN_REQUIRE(depth && dst, "resize_depth: NULL tensor pointer");
    if (int rc = check_resize("resize_depth", B, H, W, 1, fx, Ho, Wo)) return rc;
    const Mean3 m{0.0, 0.0, 0.0};
    if (depth_is_u16)
        return launch_linear<1>((const uint16_t*)depth, B, H, W, fx, Ho, Wo, m, true, (uint16_t*)dst, stream, "resize_depth");
    return launch_linear<1>((const float*)depth, B, H, W, fx, Ho, Wo, m, true, (float*)dst, stream, "resize_depth");
}

extern "C" int pcnn_resize_nearest_i32(const int32_t* label, int B, int H, int W, double fx, int Ho, int Wo, int32_t* dst, void* stream)
{
    PCNN_REQUIRE(label && dst, "resize_nearest_i32: NULL tensor pointer");
    if (int rc = check_resize("resize_nearest_i32", B, H, W, 1, fx, Ho, Wo)) return rc;
    k_resize_nearest<<<dim3(Ho, B), kThreads, 0, (cudaStream_t)stream>>>(label, H, W, 1.0 / fx, Wo, dst);
    return check_launch("resize_nearest_i32");
}
