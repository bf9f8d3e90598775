// augment.cu — the training loader's image-side augmentation on the device (lib/gt_synthesize_layer/minibatch.py:147-200,
// lib/utils/blob.py:74-129): background compositing, chromatic_transform, add_noise and the PIXEL_MEANS subtraction of the
// colour blob, and the training-time depth blob.  Every rounding is the reference's: OpenCV's uint8 HLS arithmetic (float32),
// numpy's float64 noise / clip / mean, cv2.filter2D's rounded box sum.  No operation below may be contracted into an FMA
// unless written as one, so every step is spelled with the _rn intrinsics.
#include <float.h>

#include "common.cuh"

namespace pcnn {
namespace augment {

constexpr int kTW = 64, kTH = 16, kThreads = 256;  // one CTA = a 64 x 16 tile of one image
constexpr int kHalo = 7;                           // the largest motion-blur kernel has 15 taps
constexpr int kPix = kTW * kTH / kThreads;
constexpr int kStage = (kTW + 2 * kHalo) * kTH > kTW * (kTH + 2 * kHalo) ? (kTW + 2 * kHalo) * kTH : kTW * (kTH + 2 * kHalo);

enum { kNoiseNone = 0, kNoiseGauss = 1, kNoiseBlur = 2 };

struct Params {
    int bg;        // background image, -1 = none
    int chroma;    // run chromatic_transform
    double dh, dl, ds;
    int noise;     // kNoise*
    double sigma;
    int r;         // blur radius (size = 2r + 1)
    int axis;      // 0 = along the row (x), 1 = along the column (y)
};

// A malformed table never faults: an index outside [0, n_bg) means "no background", an unknown noise mode means none, a blur
// size outside [1, 15] means 1 tap.
__device__ __forceinline__ Params load_params(const double* __restrict__ p, int n_bg)
{
    Params q;
    const double bg = p[PCNN_AUG_BACKGROUND];
    q.bg = (bg >= 0.0 && bg < (double)n_bg) ? (int)bg : -1;
    q.chroma = p[PCNN_AUG_CHROMATIC] != 0.0;
    q.dh = p[PCNN_AUG_DH];
    q.dl = p[PCNN_AUG_DL];
    q.ds = p[PCNN_AUG_DS];
    const double nm = p[PCNN_AUG_NOISE];
    q.noise = nm == 1.0 ? kNoiseGauss : nm == 2.0 ? kNoiseBlur : kNoiseNone;
    q.sigma = p[PCNN_AUG_SIGMA];
    const double sz = p[PCNN_AUG_BLUR_SIZE];
    q.r = (sz >= 1.0 && sz <= 2.0 * kHalo + 1.0) ? ((int)sz - 1) / 2 : 0;
    q.axis = p[PCNN_AUG_BLUR_AXIS] != 0.0;
    return q;
}

// Philox4x32-10 (Salmon et al., SC'11) on counter (pixel index, 0, 0, 0) and the image's 64-bit key; Box-Muller in double
// on two 53-bit uniforms: u1 in (0, 1], u2 in [0, 1).
__device__ __forceinline__ double philox_normal(uint64_t key, uint64_t pix)
{
    uint32_t w[4];
    philox4x32_10(key, pix, w);
    const uint32_t c0 = w[0], c1 = w[1], c2 = w[2], c3 = w[3];
    const double u1 = (double)(((((uint64_t)c0 << 32) | c1) >> 11) + 1) * 0x1p-53;
    const double u2 = (double)((((uint64_t)c2 << 32) | c3) >> 11) * 0x1p-53;
    return __dmul_rn(sqrt(__dmul_rn(-2.0, log(u1))), cos(__dmul_rn(6.283185307179586, u2)));
}

__device__ __forceinline__ double noise_value(const double* __restrict__ field, uint64_t key, size_t img_off, size_t pix)
{
    return field ? field[img_off + pix] : philox_normal(key, pix);
}

// np.clip keeps NaN (fminf / fmaxf would drop it)
__device__ __forceinline__ double clip255(double v) { return v < 0.0 ? 0.0 : (v > 255.0 ? 255.0 : v); }

// cv2.cvtColor(COLOR_BGR2HLS) on uint8 (RGB2HLS_b over RGB2HLS_f's vector form, OpenCV 4.x): hue = one fused multiply-add
// (x * (60 / diff) + {0 or 360 | 120 | 240}), s = diff / (l < 0.5 ? vmax + vmin : 2 - (vmax + vmin)), every output rounded
// half to even.
__device__ __forceinline__ void bgr2hls(int B8, int G8, int R8, int& H8, int& L8, int& S8)
{
    const float k = 1.f / 255.f;
    const float b = __fmul_rn((float)B8, k), g = __fmul_rn((float)G8, k), r = __fmul_rn((float)R8, k);
    const float vmax = fmaxf(fmaxf(r, g), b), vmin = fminf(fminf(r, g), b);
    const float diff = __fsub_rn(vmax, vmin), msum = __fadd_rn(vmax, vmin);
    const float l = __fmul_rn(msum, 0.5f);
    float h = 0.f, s = 0.f;
    if (diff > FLT_EPSILON) {
        s = __fdiv_rn(diff, l < 0.5f ? msum : __fsub_rn(2.f, msum));
        const float inv = __fdiv_rn(60.f, diff);
        float x, c;
        if (vmax == r) { x = __fsub_rn(g, b); c = x < 0.f ? 360.f : 0.f; }
        else if (vmax == g) { x = __fsub_rn(b, r); c = 120.f; }
        else { x = __fsub_rn(r, g); c = 240.f; }
        h = __fmaf_rn(x, inv, c);
    }
    H8 = min(255, __float2int_rn(__fmul_rn(h, 0.5f)));
    L8 = min(255, __float2int_rn(__fmul_rn(l, 255.f)));
    S8 = min(255, __float2int_rn(__fmul_rn(s, 255.f)));
}

// cv2.cvtColor(COLOR_HLS2BGR) on uint8 (HLS2RGB_b over HLS2RGB_f, hrange 180): sector table of the scalar form, outputs
// rounded half to even and saturated.
__device__ __forceinline__ void hls2bgr(int H8, int L8, int S8, int& B8, int& G8, int& R8)
{
    const float k = 1.f / 255.f;
    const float l = __fmul_rn((float)L8, k), s = __fmul_rn((float)S8, k);
    float b, g, r;
    if (s == 0.f) {
        b = g = r = l;
    } else {
        const float p2 = l <= 0.5f ? __fmul_rn(l, __fadd_rn(1.f, s)) : __fsub_rn(__fadd_rn(l, s), __fmul_rn(l, s));
        const float p1 = __fsub_rn(__fmul_rn(2.f, l), p2);
        float h = __fmul_rn((float)H8, 6.f / 180.f);
        while (h >= 6.f) h = __fsub_rn(h, 6.f);
        const int sector = (int)floorf(h);
        h = __fsub_rn(h, (float)sector);
        const float d = __fsub_rn(p2, p1);
        const float t2 = __fadd_rn(p1, __fmul_rn(d, __fsub_rn(1.f, h)));
        const float t3 = __fadd_rn(p1, __fmul_rn(d, h));
        // sector_data {1,3,0} {1,0,2} {3,0,1} {0,2,1} {0,1,3} {2,1,0} over tab = {p2, p1, t2, t3}
        switch (sector) {
            case 0: b = p1; g = t3; r = p2; break;
            case 1: b = p1; g = p2; r = t2; break;
            case 2: b = t3; g = p2; r = p1; break;
            case 3: b = p2; g = t2; r = p1; break;
            case 4: b = p2; g = p1; r = t3; break;
            default: b = t2; g = p1; r = p2; break;
        }
    }
    B8 = min(255, max(0, __float2int_rn(__fmul_rn(b, 255.f))));
    G8 = min(255, max(0, __float2int_rn(__fmul_rn(g, 255.f))));
    R8 = min(255, max(0, __float2int_rn(__fmul_rn(r, 255.f))));
}

// chromatic_transform's shifts: (h + d_h) % 180 with numpy's floor-mod, clip(l + d_l, 0, 255), then .astype('uint8')
__device__ __forceinline__ int shift_h(int h, double dh)
{
    double m = fmod(__dadd_rn((double)h, dh), 180.0);
    if (m < 0.0) m = __dadd_rn(m, 180.0);
    return (int)m;
}
__device__ __forceinline__ int shift_ls(int v, double d)
{
    const double x = __dadd_rn((double)v, d);
    return (int)(x < 0.0 ? 0.0 : (x > 255.0 ? 255.0 : x));
}

// steps 1-2 for one pixel: the composited, chromatically transformed uint8 BGR (packed b | g << 8 | r << 16)
__device__ __forceinline__ uint32_t color_px(const uint8_t* __restrict__ src, int channels, const uint8_t* __restrict__ bg_img,
                                             const Params& q, size_t pix)
{
    const uint8_t* p = src + pix * channels;
    int b = p[0], g = p[1], r = p[2];
    if (channels == 4 && p[3] == 0) {
        if (bg_img) { const uint8_t* s = bg_img + pix * 3; b = s[0]; g = s[1]; r = s[2]; }
        else b = g = r = 0;
    }
    if (q.chroma) {
        int h, l, s;
        bgr2hls(b, g, r, h, l, s);
        hls2bgr(shift_h(h, q.dh), shift_ls(l, q.dl), shift_ls(s, q.ds), b, g, r);
    }
    return (uint32_t)b | ((uint32_t)g << 8) | ((uint32_t)r << 16);
}

// reflect-101 (cv2.BORDER_DEFAULT, borderInterpolate)
__device__ __forceinline__ int reflect101(int i, int n)
{
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * n - 2 - i;
    return i;
}

// The blur tile's staging area: the tile plus kHalo pixels on each side of the blur axis, each staged pixel read at its
// reflect-101 source coordinate, so output pixel (x, y) sums staged entries (x + t, y) or (x, y + t), |t| <= r.
struct Stage {
    int sw, sh, ox, oy;  // staged extent and image coordinate of staged (0, 0)
    __device__ Stage(int axis, int x0, int y0)
    {
        sw = axis == 0 ? kTW + 2 * kHalo : kTW;
        sh = axis == 0 ? kTH : kTH + 2 * kHalo;
        ox = axis == 0 ? x0 - kHalo : x0;
        oy = axis == 0 ? y0 : y0 - kHalo;
    }
};

__global__ void __launch_bounds__(kThreads)
k_augment_color(const uint8_t* __restrict__ rgba, int channels, const uint8_t* __restrict__ bgs, int n_bg,
                const double* __restrict__ params, const uint64_t* __restrict__ keys, const double* __restrict__ field, int H, int W,
                int tiles_x, double m0, double m1, double m2, float* __restrict__ blob)
{
    __shared__ uint32_t st[kStage];
    const int b = blockIdx.y;
    const int x0 = (blockIdx.x % tiles_x) * kTW, y0 = (blockIdx.x / tiles_x) * kTH;
    const Params q = load_params(params + (size_t)b * PCNN_AUG_PARAMS, n_bg);
    const size_t img = (size_t)b * H * W;
    const uint8_t* src = rgba + img * channels;
    const uint8_t* bg_img = q.bg >= 0 ? bgs + (size_t)q.bg * H * W * 3 : nullptr;
    const uint64_t key = keys[b];
    const double mean[3] = {m0, m1, m2};

    if (q.noise == kNoiseBlur) {
        const Stage sg(q.axis, x0, y0);
        for (int i = threadIdx.x; i < sg.sw * sg.sh; i += kThreads) {
            const int sx = i % sg.sw, sy = i / sg.sw;
            const int gx = sg.ox + sx, gy = sg.oy + sy;
            if ((q.axis == 0 && gy >= H) || (q.axis == 1 && gx >= W)) continue;   // outside the image across the blur axis: unused
            st[i] = color_px(src, channels, bg_img, q, (size_t)reflect101(gy, H) * W + reflect101(gx, W));
        }
        __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < kPix; k++) {
        const int i = threadIdx.x + k * kThreads;
        const int x = x0 + i % kTW, y = y0 + i / kTW;
        if (x >= W || y >= H) continue;
        const size_t pix = (size_t)y * W + x;
        float v[3];
        if (q.noise == kNoiseBlur) {
            // round(sum / size) on the uint8 sum: size is odd, so the quotient is never a tie and this equals any accurate float sum
            const Stage sg(q.axis, x0, y0);
            const int c0 = (x - sg.ox) + (y - sg.oy) * sg.sw, step = q.axis == 0 ? 1 : sg.sw;
            int s0 = 0, s1 = 0, s2 = 0;
            for (int t = -q.r; t <= q.r; t++) {
                const uint32_t u = st[c0 + t * step];
                s0 += u & 255; s1 += (u >> 8) & 255; s2 += (u >> 16) & 255;
            }
            const int size = 2 * q.r + 1;
            v[0] = (float)((2 * s0 + size) / (2 * size));
            v[1] = (float)((2 * s1 + size) / (2 * size));
            v[2] = (float)((2 * s2 + size) / (2 * size));
        } else {
            const uint32_t u = color_px(src, channels, bg_img, q, pix);
            v[0] = (float)(u & 255); v[1] = (float)((u >> 8) & 255); v[2] = (float)((u >> 16) & 255);
            if (q.noise == kNoiseGauss) {
                const double n = __dmul_rn(q.sigma, noise_value(field, key, img, pix));   // one field for the three channels
#pragma unroll
                for (int c = 0; c < 3; c++) v[c] = __double2float_rn(clip255(__dadd_rn((double)v[c], n)));
            }
        }
        float* o = blob + (img + pix) * 3;
#pragma unroll
        for (int c = 0; c < 3; c++) o[c] = __double2float_rn(__dsub_rn((double)v[c], mean[c]));
    }
}

// per-image max(d) (numpy's im_depth_raw.max()); one CTA per image
template <typename T>
__global__ void __launch_bounds__(1024) k_depth_max(const T* __restrict__ depth, size_t hw, float* __restrict__ dmax)
{
    __shared__ float red[32];
    const T* d = depth + (size_t)blockIdx.x * hw;
    float m = -INFINITY;
    for (size_t i = threadIdx.x; i < hw; i += blockDim.x) m = fmaxf(m, (float)d[i]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = red[threadIdx.x];
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (threadIdx.x == 0) dmax[blockIdx.x] = m;
    }
}

// f32(f32(d) / max) * 255 (an all-zero image gives 0 / 0 = NaN, as numpy does)
template <typename T>
__device__ __forceinline__ float depth_px(const T* __restrict__ d, size_t pix, float mx)
{
    return __fmul_rn(__fdiv_rn((float)d[pix], mx), 255.f);
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_depth_blob(const T* __restrict__ depth, const double* __restrict__ params, const uint64_t* __restrict__ keys,
             const double* __restrict__ field, int H, int W, int tiles_x, const float* __restrict__ dmax, double m0, double m1,
             double m2, float* __restrict__ blob)
{
    __shared__ float st[kStage];
    const int b = blockIdx.y;
    const int x0 = (blockIdx.x % tiles_x) * kTW, y0 = (blockIdx.x / tiles_x) * kTH;
    const Params q = load_params(params + (size_t)b * PCNN_AUG_PARAMS, 0);
    const size_t img = (size_t)b * H * W;
    const T* d = depth + img;
    const float mx = dmax[b];
    const uint64_t key = keys[b];
    const double mean[3] = {m0, m1, m2};

    if (q.noise == kNoiseBlur) {
        const Stage sg(q.axis, x0, y0);
        for (int i = threadIdx.x; i < sg.sw * sg.sh; i += kThreads) {
            const int gx = sg.ox + i % sg.sw, gy = sg.oy + i / sg.sw;
            if ((q.axis == 0 && gy >= H) || (q.axis == 1 && gx >= W)) continue;
            st[i] = depth_px(d, (size_t)reflect101(gy, H) * W + reflect101(gx, W), mx);
        }
        __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < kPix; k++) {
        const int i = threadIdx.x + k * kThreads;
        const int x = x0 + i % kTW, y = y0 + i / kTW;
        if (x >= W || y >= H) continue;
        const size_t pix = (size_t)y * W + x;
        float v;
        if (q.noise == kNoiseBlur) {
            // the box mean on float data: the taps summed in float64 in ascending order, divided by size, rounded once
            const Stage sg(q.axis, x0, y0);
            const int c0 = (x - sg.ox) + (y - sg.oy) * sg.sw, step = q.axis == 0 ? 1 : sg.sw;
            double s = 0.0;
            for (int t = -q.r; t <= q.r; t++) s = __dadd_rn(s, (double)st[c0 + t * step]);
            v = __double2float_rn(__ddiv_rn(s, (double)(2 * q.r + 1)));
        } else {
            v = depth_px(d, pix, mx);
            if (q.noise == kNoiseGauss)
                v = __double2float_rn(clip255(__dadd_rn((double)v, __dmul_rn(q.sigma, noise_value(field, key, img, pix)))));
        }
        float* o = blob + (img + pix) * 3;
#pragma unroll
        for (int c = 0; c < 3; c++) o[c] = __double2float_rn(__dsub_rn((double)v, mean[c]));
    }
}

}  // namespace augment
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::augment;

static int check_shape(const char* what, int B, int H, int W)
{
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "%s: bad shape B=%d H=%d W=%d", what, B, H, W);
    PCNN_REQUIRE(B <= 65535, "%s: B must be <= 65535 (got %d)", what, B);
    const long long tiles = (long long)((W + kTW - 1) / kTW) * ((H + kTH - 1) / kTH);
    PCNN_REQUIRE(tiles <= 0x7fffffffLL, "%s: image too large (%d x %d)", what, H, W);
    return PCNN_OK;
}

extern "C" int pcnn_augment_color_fwd(const uint8_t* rgba, int channels, const uint8_t* backgrounds, int num_backgrounds,
                                      const double* params, const uint64_t* keys, const double* noise_field, int B, int H, int W,
                                      const double* mean3_host, float* blob, void* stream)
{
    PCNN_REQUIRE(rgba && params && keys && blob && mean3_host, "augment_color: NULL tensor pointer");
    PCNN_REQUIRE(channels == 3 || channels == 4, "augment_color: channels must be 3 or 4 (got %d)", channels);
    PCNN_REQUIRE(num_backgrounds >= 0 && (num_backgrounds == 0 || backgrounds),
                 "augment_color: num_backgrounds must be >= 0, with a background pool when > 0 (got %d)", num_backgrounds);
    if (int rc = check_shape("augment_color", B, H, W)) return rc;
    const int tiles_x = (W + kTW - 1) / kTW, tiles = tiles_x * ((H + kTH - 1) / kTH);
    k_augment_color<<<dim3(tiles, B), kThreads, 0, (cudaStream_t)stream>>>(rgba, channels, backgrounds, num_backgrounds, params, keys,
                                                                          noise_field, H, W, tiles_x, mean3_host[0], mean3_host[1],
                                                                          mean3_host[2], blob);
    return check_launch("augment_color");
}

extern "C" int pcnn_depth_blob_train_fwd(const void* depth, int depth_is_u16, const double* params, const uint64_t* keys,
                                         const double* noise_field, int B, int H, int W, const double* mean3_host, float* depth_max,
                                         float* blob, void* stream)
{
    PCNN_REQUIRE(depth && params && keys && depth_max && blob && mean3_host, "depth_blob_train: NULL tensor pointer");
    if (int rc = check_shape("depth_blob_train", B, H, W)) return rc;
    const int tiles_x = (W + kTW - 1) / kTW, tiles = tiles_x * ((H + kTH - 1) / kTH);
    const size_t hw = (size_t)H * W;
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid(tiles, B);
    if (depth_is_u16) {
        const uint16_t* d = (const uint16_t*)depth;
        k_depth_max<uint16_t><<<B, 1024, 0, s>>>(d, hw, depth_max);
        k_depth_blob<uint16_t><<<grid, kThreads, 0, s>>>(d, params, keys, noise_field, H, W, tiles_x, depth_max, mean3_host[0],
                                                         mean3_host[1], mean3_host[2], blob);
    } else {
        const float* d = (const float*)depth;
        k_depth_max<float><<<B, 1024, 0, s>>>(d, hw, depth_max);
        k_depth_blob<float><<<grid, kThreads, 0, s>>>(d, params, keys, noise_field, H, W, tiles_x, depth_max, mean3_host[0],
                                                      mean3_host[1], mean3_host[2], blob);
    }
    return check_launch("depth_blob_train");
}
