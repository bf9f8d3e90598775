// coord_pose.cu — pose estimation from predicted object coordinates (DESIGN.md §13), the device counterpart of the reference's
// Synthesizer::estimatePose3D (lib/synthesize/synthesize.cpp:1769-1966): preemptive RANSAC over camera-point / object-coordinate
// correspondences, Kabsch refinement, a bounded Nelder-Mead polish of the survivor; and of the colour-only
// Synthesizer::estimatePose2D (:1571-1767): preemptive RANSAC over pixel / object-coordinate correspondences with P3P hypotheses.
//
//   k_lists    one CTA per image: per-class pixel lists in the reference's column-major order (x outer, y inner), two passes
//              over warp-owned segments of that order (warp-aggregated counts, then ranked scatter); a depth hole is flagged in
//              bit 31 of the list entry (with depth only)
//   k_sample   one CTA per image, thread h = hypothesis h: draws (object, three pixels) until samplePoint3D, Kabsch, the
//              reconstruction check and the projected-box area all pass, at most kMaxAttempts times
//   k_sample2d one warp per hypothesis, lane i = attempt base + i: (object, four pixels), samplePoint2D, the point-line checks,
//              P3P, the 10 px reconstruction and the projected-box area; a ballot keeps the lowest accepted attempt
//   k_ransac   one CTA per (class, image): the preemptive loop (warp 0 walks the pixel subset of the round, one warp per
//              hypothesis counts inliers with ballots, rank selection keeps the better half, one warp per survivor refits
//              with Kabsch), then Nelder-Mead on the survivor with the block evaluating the energy; the colour-only
//              instantiation counts with the reprojection gate and neither refits nor polishes
// Random numbers are Philox4x32-10 on the image's key with counters that name the draw (stream, hypothesis / class, round,
// index), so an image's result depends on its own inputs and key only.  Every reduction has a fixed order.
#include <cuda_runtime.h>
#include <limits.h>

#include <type_traits>

#include "common.cuh"
#include "heads_common.cuh"
#include "pose_common.cuh"

namespace pcnn {
namespace coordpose {

constexpr int kHyp = 256;            // ransacIterations
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kRounds = 8;           // refIt: with <= 256 hypotheses per object every object stops after exactly 8 rounds
constexpr int kBatch = 1000;         // preemptiveBatch
constexpr int kMaxInl = 1000;        // maxPixels of filterInliers3D
constexpr int kMinFinal = 10;        // minPixels: Nelder-Mead only above this many inliers
constexpr int kMinArea = 400;        // minArea: object pixels and projected-box area
constexpr int kMaxTaken = 12288;     // pixels one round can take (expected at most ~10.7k, see DESIGN §13)
constexpr int kWords = kMaxTaken / 32;
constexpr int kMaxAttempts = 1024;   // the reference tries up to 10^7 times per hypothesis
constexpr int kNMEvals = 100;        // refinementIterations
constexpr int kListThreads = 1024;
constexpr int kRecThreads = 256;
constexpr int kMaxC = 128;
constexpr int kInfo = 6;
constexpr int kTraceHyp = 5 + kRounds, kTraceRound = 4;   // per hypothesis: class, attempts, triple, count per round
constexpr int kTraceHyp2D = 6 + kRounds;                   // colour-only: class, attempts, four pixels, count per round
constexpr int kSampleWarps = 8;                             // k_sample2d: one warp per hypothesis
constexpr uint32_t kHole = 0x80000000u;
constexpr double kGate = (double)0.01f;        // inlierThreshold3D = minDist3D = 0.01f
constexpr double kGate2D = 10.0;               // inlierThreshold2D = minDist2D = 10 px
constexpr double kRankTol = 1e-6;              // second singular value <= kRankTol * first: collinear, no unique rotation
constexpr int kBisect = 200;                   // bisection steps per polynomial root (about 64 reach the last bit near 1)

struct Hyp {
    double R[9], t[3];
    int obj, attempts;
};

struct Args {
    const int32_t* label;
    const float* depth;
    const float* dense;     // [B,H,W,3C] or NULL
    const float* lowres;    // [B,H/8,W/8,4C] (with dense == NULL)
    const float* bias;      // [3C]
    const float* meta;
    const float* ext;
    const uint64_t* keys;
    int num_meta, B, H, W, C;
    float factor;
    const int* counts;
    const int* start;
    const int* list;
    const int* exhausted;
    Hyp* hyps;
    int* taken;
    float* teye;
    float* tobj;
    float* poses;
    float* info;
    int32_t* trace_hyp;
    int32_t* trace_round;
};

__device__ __forceinline__ uint64_t ctr_hyp(int h, int att) { return (1ull << 60) | ((uint64_t)h << 32) | (uint32_t)att; }
__device__ __forceinline__ uint64_t ctr_sub(int c, int r, uint64_t k) { return (2ull << 60) | ((uint64_t)c << 48) | ((uint64_t)r << 40) | k; }
__device__ __forceinline__ uint64_t ctr_fil(int h, int r, int j) { return (3ull << 60) | ((uint64_t)h << 48) | ((uint64_t)r << 40) | (uint32_t)j; }
// colour-only attempts: word 0 = object, words 1-3 = pixels 1-3 / word 0 = pixel 4
__device__ __forceinline__ uint64_t ctr_p2a(int h, int att) { return (4ull << 60) | ((uint64_t)h << 32) | (uint32_t)att; }
__device__ __forceinline__ uint64_t ctr_p2b(int h, int att) { return (5ull << 60) | ((uint64_t)h << 32) | (uint32_t)att; }
__device__ __forceinline__ int uniform_int(uint32_t w, int n) { return (int)(((uint64_t)w * (uint32_t)n) >> 32); }

// camera point of pixel idx (pxToEye, synthesize.cpp:1372-1389), float, in the reference's operation order
__device__ __forceinline__ float3 eye_at(const float* depth, int W, float fx, float fy, float px, float py, float factor, int idx)
{
    const int x = idx % W, y = idx / W;
    const float d = __ldg(depth + idx);
    return make_float3(__fdiv_rn(__fdiv_rn(__fmul_rn(__fsub_rn((float)x, px), d), fx), factor),
                       __fdiv_rn(__fdiv_rn(__fmul_rn(__fsub_rn((float)y, py), d), fy), factor), __fdiv_rn(d, factor));
}

// object coordinate of class c at pixel idx of image b (getMode3D, :1051-1072): a, b formed in double and rounded to float
__device__ __forceinline__ float3 mode_at(const Args& a, int b, int c, int idx)
{
    const int x = idx % a.W, y = idx / a.W;
    float v[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float raw = a.dense ? __ldg(a.dense + ((size_t)b * a.H * a.W + idx) * 3 * a.C + 3 * c + k)
                                  : up8_value(a.lowres, b, a.H / 8, a.W / 8, 4 * a.C, a.C + 3 * c + k, y, x, __ldg(a.bias + 3 * c + k));
        const float e = __ldg(a.ext + 3 * c + k);
        const float vmin = __fdiv_rn(-e, 2.f), vmax = __fdiv_rn(e, 2.f);
        const float den = __fsub_rn(vmax, vmin);
        const float sa = (float)__ddiv_rn(1.0, (double)den);
        const float sb = (float)__ddiv_rn(__dmul_rn(-1.0, (double)vmin), (double)den);
        v[k] = __fdiv_rn(__fsub_rn(raw, sb), sa);
    }
    return make_float3(v[0], v[1], v[2]);
}

// cv::norm of a float point difference: float subtraction, double sum of squares
__device__ __forceinline__ double dist_f(float3 p, float3 q)
{
    const float dx = __fsub_rn(p.x, q.x), dy = __fsub_rn(p.y, q.y), dz = __fsub_rn(p.z, q.z);
    return sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

__device__ __forceinline__ double3 xform(const double* R, const double* t, double x, double y, double z)
{
    return make_double3(R[0] * x + R[1] * y + R[2] * z + t[0], R[3] * x + R[4] * y + R[5] * z + t[1],
                        R[6] * x + R[7] * y + R[8] * z + t[2]);
}

__device__ __forceinline__ bool is_inlier(const double* R, const double* t, float3 e, float3 o)
{
    const double3 q = xform(R, t, o.x, o.y, o.z);
    const double dx = e.x - q.x, dy = e.y - q.y, dz = e.z - q.z;
    return sqrt(dx * dx + dy * dy + dz * dz) < kGate;
}

// cv::projectPoints of one object point (double): x / z, y / z (z = 0 taken as 1), then the intrinsics
__device__ __forceinline__ double2 project(const double* R, const double* t, const double* cam, double X, double Y, double Z)
{
    const double3 q = xform(R, t, X, Y, Z);
    const double iz = q.z != 0.0 ? 1.0 / q.z : 1.0;
    return make_double2(q.x * iz * cam[0] + cam[2], q.y * iz * cam[1] + cam[3]);
}

// the inlier tests of the preemptive loop: e is the taken pixel's camera point (3-D) or its pixel (x, y, 0) (2-D)
struct Gate3D {             // countInliers3D: within 1 cm of R o + t
    __device__ Gate3D(float, float, float, float) {}
    __device__ bool operator()(const double* R, const double* t, float3 e, float3 o) const { return is_inlier(R, t, e, o); }
};
struct Gate2D {             // countInliers2D: within 10 px of the projection of o
    double cam[4];          // fx, fy, px, py
    __device__ Gate2D(float fx, float fy, float px, float py) : cam{fx, fy, px, py} {}
    __device__ bool operator()(const double* R, const double* t, float3 e, float3 o) const
    {
        const double2 q = project(R, t, cam, o.x, o.y, o.z);
        const double dx = (double)e.x - q.x, dy = (double)e.y - q.y;
        return sqrt(dx * dx + dy * dy) < kGate2D;
    }
};

// Kabsch (Hypothesis::calcRigidBodyTransform, Hypothesis.cpp:217-241) on the covariance a = sum (A - cA)(B - cB)^T:
// a = U S V^T by one-sided Jacobi, R = V diag(1, 1, det(V U^T)) U^T, t = cB - R cA.  U's third column is completed as
// u1 x u2: the product d * v3 u3^T does not depend on that sign.  False when a is (numerically) of rank < 2.
__device__ bool kabsch(const double* a, const double* cA, const double* cB, double* R, double* t)
{
    double G[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int k = 0; k < 9; k++) G[k] = a[k];
    for (int sweep = 0; sweep < 30; sweep++) {
        bool rotated = false;
        for (int p = 0; p < 2; p++)
            for (int q = p + 1; q < 3; q++) {
                double al = 0, be = 0, ga = 0;
                for (int i = 0; i < 3; i++) {
                    al += G[3 * i + p] * G[3 * i + p];
                    be += G[3 * i + q] * G[3 * i + q];
                    ga += G[3 * i + p] * G[3 * i + q];
                }
                if (!(fabs(ga) > 1e-17 * sqrt(al * be))) continue;
                rotated = true;
                const double zeta = (be - al) / (2.0 * ga);
                const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + tt * tt), s = c * tt;
                for (int i = 0; i < 3; i++) {
                    const double gp = G[3 * i + p], gq = G[3 * i + q];
                    G[3 * i + p] = c * gp - s * gq;
                    G[3 * i + q] = s * gp + c * gq;
                    const double vp = V[3 * i + p], vq = V[3 * i + q];
                    V[3 * i + p] = c * vp - s * vq;
                    V[3 * i + q] = s * vp + c * vq;
                }
            }
        if (!rotated) break;
    }
    double sv[3];
    int ord[3] = {0, 1, 2};
    for (int k = 0; k < 3; k++) sv[k] = sqrt(G[k] * G[k] + G[3 + k] * G[3 + k] + G[6 + k] * G[6 + k]);
    for (int i = 0; i < 2; i++)         // descending singular values
        for (int j = 0; j < 2 - i; j++)
            if (sv[ord[j]] < sv[ord[j + 1]]) { const int tmp = ord[j]; ord[j] = ord[j + 1]; ord[j + 1] = tmp; }
    const double s0 = sv[ord[0]], s1 = sv[ord[1]];
    if (!(s0 > 0.0) || !(s1 > kRankTol * s0) || !isfinite(s0)) return false;
    double U[3][3], Vs[3][3];           // columns
    for (int k = 0; k < 2; k++)
        for (int i = 0; i < 3; i++) U[k][i] = G[3 * i + ord[k]] / sv[ord[k]];
    U[2][0] = U[0][1] * U[1][2] - U[0][2] * U[1][1];
    U[2][1] = U[0][2] * U[1][0] - U[0][0] * U[1][2];
    U[2][2] = U[0][0] * U[1][1] - U[0][1] * U[1][0];
    for (int k = 0; k < 3; k++)
        for (int i = 0; i < 3; i++) Vs[k][i] = V[3 * i + ord[k]];
    const double detV = Vs[0][0] * (Vs[1][1] * Vs[2][2] - Vs[1][2] * Vs[2][1]) - Vs[1][0] * (Vs[0][1] * Vs[2][2] - Vs[0][2] * Vs[2][1]) +
                        Vs[2][0] * (Vs[0][1] * Vs[1][2] - Vs[0][2] * Vs[1][1]);
    const double d = detV < 0 ? -1.0 : 1.0;     // det(U) = +1 by construction
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) R[3 * i + j] = Vs[0][i] * U[0][j] + Vs[1][i] * U[1][j] + d * Vs[2][i] * U[2][j];
    for (int i = 0; i < 3; i++) t[i] = cB[i] - (R[3 * i] * cA[0] + R[3 * i + 1] * cA[1] + R[3 * i + 2] * cA[2]);
    return true;
}

// cv::Rodrigues, vector -> matrix and matrix -> vector (double)
__device__ void rodrigues_exp(const double* r, double* R)
{
    const double th = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    if (th < 2.220446049250313e-16) {
        for (int k = 0; k < 9; k++) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
        return;
    }
    const double c = cos(th), s = sin(th), c1 = 1.0 - c, x = r[0] / th, y = r[1] / th, z = r[2] / th;
    R[0] = c + c1 * x * x;     R[1] = c1 * x * y - s * z; R[2] = c1 * x * z + s * y;
    R[3] = c1 * x * y + s * z; R[4] = c + c1 * y * y;     R[5] = c1 * y * z - s * x;
    R[6] = c1 * x * z - s * y; R[7] = c1 * y * z + s * x; R[8] = c + c1 * z * z;
}

__device__ void rodrigues_log(const double* R, double* r)
{
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1.0) * 0.5;
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    double th = acos(c);
    if (s < 1e-5) {
        if (c > 0) { r[0] = r[1] = r[2] = 0.0; return; }
        rx = sqrt(fmax((R[0] + 1.0) * 0.5, 0.0));
        ry = sqrt(fmax((R[4] + 1.0) * 0.5, 0.0)) * (R[1] < 0 ? -1.0 : 1.0);
        rz = sqrt(fmax((R[8] + 1.0) * 0.5, 0.0)) * (R[2] < 0 ? -1.0 : 1.0);
        if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && ((R[5] > 0) != (ry * rz > 0))) rz = -rz;
        th /= sqrt(rx * rx + ry * ry + rz * rz);
        r[0] = rx * th; r[1] = ry * th; r[2] = rz * th;
        return;
    }
    const double v = th / (2.0 * s);
    r[0] = rx * v; r[1] = ry * v; r[2] = rz * v;
}

// float -> int as the reference's `int = float` compiles on x86-64 (cvttss2si): truncation, and INT_MIN for anything outside
// the int range (NaN never reaches it: std::min / std::max keep the int side)
__device__ __forceinline__ int f2i_x86(float v) { return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }

// area of getBB2D (detection.h:78-109) of the class's 3-D box under (R, t)
__device__ int bb_area(const float* e, const double* R, const double* t, float fx, float fy, float px, float py, int W, int H)
{
    const float hx = __fdiv_rn(e[0], 2.f), hy = __fdiv_rn(e[1], 2.f), hz = __fdiv_rn(e[2], 2.f);
    int minX = W - 1, maxX = 0, minY = H - 1, maxY = 0;
    for (int k = 0; k < 8; k++) {
        const double X = (k & 4) ? -hx : hx, Y = (k & 2) ? -hy : hy, Z = (k & 1) ? -hz : hz;
        const double3 q = xform(R, t, X, Y, Z);
        const double iz = q.z != 0.0 ? 1.0 / q.z : 1.0;
        const float u = (float)(q.x * iz * (double)fx + (double)px), v = (float)(q.y * iz * (double)fy + (double)py);
        minX = f2i_x86(u < (float)minX ? u : (float)minX);
        minY = f2i_x86(v < (float)minY ? v : (float)minY);
        maxX = f2i_x86((float)maxX < u ? u : (float)maxX);
        maxY = f2i_x86((float)maxY < v ? v : (float)maxY);
    }
    minX = min(max(minX, 0), W - 1); maxX = min(max(maxX, 0), W - 1);
    minY = min(max(minY, 0), H - 1); maxY = min(max(maxY, 0), H - 1);
    return (maxX - minX + 1) * (maxY - minY + 1);
}

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------------- pixel lists
// kDepth = false (the colour-only estimator): no depth, no hole bit
template <bool kDepth>
__global__ void __launch_bounds__(kListThreads)
k_lists(const int32_t* __restrict__ label, const float* __restrict__ depth, int H, int W, int C, int* __restrict__ counts,
        int* __restrict__ start, int* __restrict__ list)
{
    __shared__ int cnt[32][kMaxC];
    __shared__ int cstart[kMaxC];
    const int b = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int HW = H * W;
    const int32_t* L = label + (size_t)b * HW;
    const float* D = kDepth ? depth + (size_t)b * HW : nullptr;
    for (int i = threadIdx.x; i < 32 * kMaxC; i += kListThreads) (&cnt[0][0])[i] = 0;
    __syncthreads();
    const int seg = (HW + 31) / 32, lo = w * seg, hi = min(HW, lo + seg);
    for (int base = lo; base < hi; base += 32) {
        const int i = base + lane;           // column-major position: x = i / H, y = i % H
        const int l0 = i < hi ? __ldg(L + (size_t)(i % H) * W + i / H) : -1;
        const int l = (l0 >= 0 && l0 < C) ? l0 : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, l);
        if (l >= 0 && lane == __ffs(peers) - 1) cnt[w][l] += __popc(peers);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int c = 0; c < C; c++) {
            int n = 0;
            for (int k = 0; k < 32; k++) n += cnt[k][c];
            cstart[c] = acc;
            counts[(size_t)b * C + c] = n;
            start[(size_t)b * C + c] = acc;
            acc += n;
        }
    }
    __syncthreads();
    if (threadIdx.x < C) {
        int run = cstart[threadIdx.x];
        for (int k = 0; k < 32; k++) { const int n = cnt[k][threadIdx.x]; cnt[k][threadIdx.x] = run; run += n; }
    }
    __syncthreads();
    int* out = list + (size_t)b * HW;
    for (int base = lo; base < hi; base += 32) {
        const int i = base + lane;
        const int idx = i < hi ? (i % H) * W + i / H : 0;
        const int l0 = i < hi ? __ldg(L + idx) : -1;
        const int l = (l0 >= 0 && l0 < C) ? l0 : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, l);
        if (l >= 0) out[cnt[w][l] + __popc(peers & ((1u << lane) - 1u))] = idx | ((kDepth && __ldg(D + idx) == 0.f) ? (int)kHole : 0);
        __syncwarp();
        if (l >= 0 && lane == __ffs(peers) - 1) cnt[w][l] += __popc(peers);
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------- hypotheses
__global__ void __launch_bounds__(kHyp)
k_sample(const Args a, int* __restrict__ exhausted)
{
    __shared__ int objs[kMaxC];
    __shared__ int nobj;
    const int b = blockIdx.x, h = threadIdx.x;
    const int* counts = a.counts + (size_t)b * a.C;
    if (h == 0) {
        int n = 0;
        for (int c = 1; c < a.C; c++)
            if (counts[c] > kMinArea) objs[n++] = c;
        nobj = n;
    }
    __syncthreads();
    Hyp& out = a.hyps[(size_t)b * kHyp + h];
    int32_t* tr = a.trace_hyp ? a.trace_hyp + ((size_t)b * kHyp + h) * kTraceHyp : nullptr;
    const float* m = a.meta + (size_t)b * a.num_meta;
    const float fx = m[0], px = m[2], fy = m[4], py = m[5];
    const int HW = a.H * a.W;
    const uint64_t key = a.keys[b];
    bool found = false;
    int att = 0, obj = 0, pix[3] = {0, 0, 0};
    if (nobj > 0) {
        for (; att < kMaxAttempts && !found; att++) {
            uint32_t w[4];
            philox4x32_10(key, ctr_hyp(h, att), w);
            obj = objs[uniform_int(w[0], nobj)];
            const int N = counts[obj];
            const int* L = a.list + (size_t)b * HW + a.start[(size_t)b * a.C + obj];
            float3 eye[3], oc[3];
            bool ok = true;
            for (int k = 0; k < 3 && ok; k++) {
                const int entry = __ldg(L + uniform_int(w[k + 1], N));
                pix[k] = entry & ~(int)kHole;
                if (entry & (int)kHole) { ok = false; break; }           // depth hole
                eye[k] = eye_at(a.depth + (size_t)b * HW, a.W, fx, fy, px, py, a.factor, pix[k]);
                double md = -1.0;
                for (int j = 0; j < k; j++) { const double d = dist_f(eye[j], eye[k]); md = md < 0 ? d : fmin(md, d); }
                if (md > 0 && md < kGate) { ok = false; break; }
                oc[k] = mode_at(a, b, obj, pix[k]);
                if (oc[k].x == 0.f && oc[k].y == 0.f && oc[k].z == 0.f) { ok = false; break; }   // empty prediction
                md = -1.0;
                for (int j = 0; j < k; j++) { const double d = dist_f(oc[j], oc[k]); md = md < 0 ? d : fmin(md, d); }
                if (md > 0 && md < kGate) { ok = false; break; }
            }
            if (!ok) continue;
            double cA[3] = {0, 0, 0}, cB[3] = {0, 0, 0};
            for (int k = 0; k < 3; k++) {
                cA[0] += oc[k].x; cA[1] += oc[k].y; cA[2] += oc[k].z;
                cB[0] += eye[k].x; cB[1] += eye[k].y; cB[2] += eye[k].z;
            }
            for (int i = 0; i < 3; i++) { cA[i] *= 1.0 / 3.0; cB[i] *= 1.0 / 3.0; }
            double cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            for (int k = 0; k < 3; k++) {
                const double pa[3] = {oc[k].x - cA[0], oc[k].y - cA[1], oc[k].z - cA[2]};
                const double pb[3] = {eye[k].x - cB[0], eye[k].y - cB[1], eye[k].z - cB[2]};
                for (int i = 0; i < 3; i++)
                    for (int j = 0; j < 3; j++) cov[3 * i + j] += pa[i] * pb[j];
            }
            if (!kabsch(cov, cA, cB, out.R, out.t)) continue;                     // collinear triple
            bool recon = true;
            for (int k = 0; k < 3; k++) recon = recon && is_inlier(out.R, out.t, eye[k], oc[k]);
            if (!recon) continue;
            if (bb_area(a.ext + 3 * obj, out.R, out.t, fx, fy, px, py, a.W, a.H) < kMinArea) continue;
            found = true;
        }
    }
    out.obj = found ? obj : 0;
    out.attempts = att;
    if (tr) {
        tr[0] = found ? obj : 0; tr[1] = att;
        for (int k = 0; k < 3; k++) tr[2 + k] = found ? pix[k] : -1;
        for (int r = 0; r < kRounds; r++) tr[5 + r] = -1;
    }
    const int n_ex = __syncthreads_count(nobj > 0 && !found);
    if (h == 0) exhausted[b] = n_ex;
}

// ------------------------------------------------------------------------------------------------- colour-only hypotheses
// The polynomial arithmetic rounds every step (no contraction), as tests/coord_pose2d_ref.py does in Python floats.
__device__ __forceinline__ double horner(const double* c, int n, double x)     // c[0] x^n + ... + c[n]
{
    double v = c[0];
    for (int i = 1; i <= n; i++) v = __dadd_rn(__dmul_rn(v, x), c[i]);
    return v;
}

// the root of c in (lo, hi), f(lo) = flo of the opposite sign to f(hi), bisected until the midpoint is an end point
__device__ double bisect(const double* c, int n, double lo, double hi, double flo)
{
    double mid = __dmul_rn(0.5, __dadd_rn(lo, hi));
    for (int it = 0; it < kBisect && mid > lo && mid < hi; it++) {
        const double fm = horner(c, n, mid);
        if (fm == 0.0) return mid;
        if ((fm < 0.0) == (flo < 0.0)) { lo = mid; flo = fm; } else hi = mid;
        mid = __dmul_rn(0.5, __dadd_rn(lo, hi));
    }
    return mid;
}

// real roots of the monic quartic x^4 + p[0] x^3 + p[1] x^2 + p[2] x + p[3], ascending.  The roots of each derivative split
// [-bound, bound] (Cauchy's bound, which holds the derivatives' roots too by Gauss-Lucas) into brackets of the next lower
// derivative; a bracket whose ends differ in sign holds one root.  A root of even multiplicity has no sign change and is missed.
__device__ int quartic_roots(const double* p, double* x)
{
    double bound = 1.0;
    for (int i = 0; i < 4; i++) bound = fmax(bound, 1.0 + fabs(p[i]));
    const double c[3][5] = {{6.0, 3.0 * p[0], p[1]}, {4.0, 3.0 * p[0], 2.0 * p[1], p[2]}, {1.0, p[0], p[1], p[2], p[3]}};
    double r[4] = {-p[0] / 4.0};
    int n = 1;
    for (int deg = 2; deg <= 4; deg++) {
        const double* cc = c[deg - 2];
        double nr[4], lo = -bound, flo = horner(cc, deg, lo);
        int m = 0;
        for (int i = 0; i <= n; i++) {
            const double hi = i < n ? fmin(fmax(r[i], -bound), bound) : bound, fhi = horner(cc, deg, hi);
            if (flo != 0.0 && fhi != 0.0 && (flo < 0.0) != (fhi < 0.0) && lo < hi) nr[m++] = bisect(cc, deg, lo, hi, flo);
            lo = hi;
            flo = fhi;
        }
        for (int i = 0; i < m; i++) r[i] = nr[i];
        n = m;
    }
    for (int i = 0; i < n; i++) x[i] = r[i];
    return n;
}

// P3P (cv::solvePnP with SOLVEPNP_P3P): Grunert's quartic in v = s3 / s1 (Haralick et al., "Review and analysis of solutions of
// the three point perspective pose estimation problem", IJCV 1994, eqs. 8-9) on the first three correspondences.  Every positive
// real root gives the distances s1, s2 = u s1, s3 = v s1 along the bearing rays and the pose by Kabsch on the three camera
// points; the root whose pose reprojects the fourth point closest (first root on a tie) wins.  False when no root gives a pose.
// Up to the Kabsch step every operation rounds on its own, in tests/coord_pose2d_ref.py's order of evaluation: for a small object
// far from the camera the roots cluster near v = 1 and a last-bit change of a coefficient moves them by ~1e-4.
__device__ bool p3p(const float3* o, const float* pu, const float* pv, const double* cam, double* R, double* t)
{
    const auto mu = [](double x, double y) { return __dmul_rn(x, y); };
    const auto ad = [](double x, double y) { return __dadd_rn(x, y); };
    const auto sb = [](double x, double y) { return __dsub_rn(x, y); };
    const auto dv = [](double x, double y) { return __ddiv_rn(x, y); };
    double f[3][3], P[3][3];
    for (int k = 0; k < 3; k++) {
        const double xn = dv(sb(pu[k], cam[2]), cam[0]), yn = dv(sb(pv[k], cam[3]), cam[1]);
        const double nn = sqrt(ad(ad(mu(xn, xn), mu(yn, yn)), 1.0));
        f[k][0] = dv(xn, nn); f[k][1] = dv(yn, nn); f[k][2] = dv(1.0, nn);
        P[k][0] = o[k].x; P[k][1] = o[k].y; P[k][2] = o[k].z;
    }
    auto sq = [&](int i, int j) {
        const double dx = sb(P[i][0], P[j][0]), dy = sb(P[i][1], P[j][1]), dz = sb(P[i][2], P[j][2]);
        return ad(ad(mu(dx, dx), mu(dy, dy)), mu(dz, dz));
    };
    auto dot = [&](int i, int j) { return ad(ad(mu(f[i][0], f[j][0]), mu(f[i][1], f[j][1])), mu(f[i][2], f[j][2])); };
    const double a2 = sq(1, 2), b2 = sq(0, 2), c2 = sq(0, 1);
    if (!(b2 > 0.0)) return false;
    const double ca = dot(1, 2), cb = dot(0, 2), cg = dot(0, 1);
    const double amc = dv(sb(a2, c2), b2), apc = dv(ad(a2, c2), b2);
    const double A4 = sb(mu(sb(amc, 1.0), sb(amc, 1.0)), mu(mu(dv(mu(4.0, c2), b2), ca), ca));
    const double A3 = mu(4.0, ad(sb(mu(mu(amc, sb(1.0, amc)), cb), mu(mu(sb(1.0, apc), ca), cg)), mu(mu(mu(dv(mu(2.0, c2), b2), ca), ca), cb)));
    const double A2 = mu(2.0, ad(sb(ad(ad(sb(mu(amc, amc), 1.0), mu(mu(mu(mu(2.0, amc), amc), cb), cb)), mu(mu(dv(mu(2.0, sb(b2, c2)), b2), ca), ca)),
                                    mu(mu(mu(mu(4.0, apc), ca), cb), cg)),
                                 mu(mu(dv(mu(2.0, sb(b2, a2)), b2), cg), cg)));
    const double A1 = mu(4.0, sb(ad(mu(mu(-amc, ad(1.0, amc)), cb), mu(mu(mu(dv(mu(2.0, a2), b2), cg), cg), cb)), mu(mu(sb(1.0, apc), ca), cg)));
    const double A0 = sb(mu(ad(1.0, amc), ad(1.0, amc)), mu(mu(dv(mu(4.0, a2), b2), cg), cg));
    const double p[4] = {dv(A3, A4), dv(A2, A4), dv(A1, A4), dv(A0, A4)};
    if (!(A4 != 0.0) || !isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2]) || !isfinite(p[3])) return false;
    double v[4];
    const int nv = quartic_roots(p, v);
    double best = INFINITY;
    for (int i = 0; i < nv; i++) {
        const double den = mu(2.0, sb(cg, mu(v[i], ca)));
        if (!(v[i] > 0.0) || den == 0.0) continue;
        const double u = dv(ad(ad(sb(mu(mu(sb(amc, 1.0), v[i]), v[i]), mu(mu(mu(2.0, amc), cb), v[i])), 1.0), amc), den);
        const double s1q = dv(b2, sb(ad(1.0, mu(v[i], v[i])), mu(mu(2.0, v[i]), cb)));
        if (!(u > 0.0) || !(s1q > 0.0) || !isfinite(s1q)) continue;
        const double s[3] = {sqrt(s1q), mu(u, sqrt(s1q)), mu(v[i], sqrt(s1q))};
        double cA[3] = {0, 0, 0}, cB[3] = {0, 0, 0}, X[3][3];
        for (int k = 0; k < 3; k++)
            for (int d = 0; d < 3; d++) { X[k][d] = mu(s[k], f[k][d]); cA[d] += P[k][d]; cB[d] += X[k][d]; }
        for (int d = 0; d < 3; d++) { cA[d] *= 1.0 / 3.0; cB[d] *= 1.0 / 3.0; }
        double cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, Ri[9], ti[3];
        for (int k = 0; k < 3; k++)
            for (int x = 0; x < 3; x++)
                for (int y = 0; y < 3; y++) cov[3 * x + y] += (P[k][x] - cA[x]) * (X[k][y] - cB[y]);
        if (!kabsch(cov, cA, cB, Ri, ti)) continue;
        const double2 q = project(Ri, ti, cam, o[3].x, o[3].y, o[3].z);
        const double dx = pu[3] - q.x, dy = pv[3] - q.y, err = sqrt(dx * dx + dy * dy);
        if (err < best) {
            best = err;
            for (int k = 0; k < 9; k++) R[k] = Ri[k];
            for (int k = 0; k < 3; k++) t[k] = ti[k];
        }
    }
    return best < INFINITY;
}

// pointLineDistance (synthesize.cpp:1077-1083): |(q - p) x (r - p)| / |q - p| with float differences and cross product
__device__ __forceinline__ double line_dist(float3 p, float3 q, float3 r)
{
    const float ax = __fsub_rn(q.x, p.x), ay = __fsub_rn(q.y, p.y), az = __fsub_rn(q.z, p.z);
    const float bx = __fsub_rn(r.x, p.x), by = __fsub_rn(r.y, p.y), bz = __fsub_rn(r.z, p.z);
    const float cx = __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by)), cy = __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz)),
                cz = __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx));
    const double nc = sqrt((double)cx * cx + (double)cy * cy + (double)cz * cz), na = sqrt((double)ax * ax + (double)ay * ay + (double)az * az);
    return nc / na;
}

// one attempt of estimatePose2D's sampling loop (synthesize.cpp:1616-1690): object, four samplePoint2D pixels, the four
// point-line checks, P3P, the reconstruction of all four within 10 px (float projections) and the projected-box area
__device__ bool attempt2d(const Args& a, int b, const int* objs, int nobj, const double* cam, uint64_t key, int h, int att,
                          double* R, double* t, int& obj, int* pix)
{
    uint32_t w0[4], w1[4];
    philox4x32_10(key, ctr_p2a(h, att), w0);
    philox4x32_10(key, ctr_p2b(h, att), w1);
    obj = objs[uniform_int(w0[0], nobj)];
    const int N = a.counts[(size_t)b * a.C + obj];
    const int* L = a.list + (size_t)b * a.H * a.W + a.start[(size_t)b * a.C + obj];
    float3 oc[4];
    float pu[4], pv[4];
    for (int k = 0; k < 4; k++) {
        pix[k] = __ldg(L + uniform_int(k < 3 ? w0[k + 1] : w1[0], N));
        pu[k] = (float)(pix[k] % a.W);
        pv[k] = (float)(pix[k] / a.W);
        double md = -1.0;
        for (int j = 0; j < k; j++) {
            const float dx = __fsub_rn(pu[j], pu[k]), dy = __fsub_rn(pv[j], pv[k]);
            const double d = sqrt((double)dx * dx + (double)dy * dy);
            md = md < 0 ? d : fmin(md, d);
        }
        if (md > 0 && md < kGate2D) return false;
        oc[k] = mode_at(a, b, obj, pix[k]);
        if (oc[k].x == 0.f && oc[k].y == 0.f && oc[k].z == 0.f) return false;      // empty prediction
        md = -1.0;
        for (int j = 0; j < k; j++) { const double d = dist_f(oc[j], oc[k]); md = md < 0 ? d : fmin(md, d); }
        if (md > 0 && md < kGate) return false;
    }
    if (line_dist(oc[0], oc[1], oc[2]) < kGate || line_dist(oc[0], oc[1], oc[3]) < kGate || line_dist(oc[0], oc[2], oc[3]) < kGate ||
        line_dist(oc[1], oc[2], oc[3]) < kGate)
        return false;                                                          // NaN (coincident points) passes, as in the reference
    if (!p3p(oc, pu, pv, cam, R, t)) return false;
    for (int k = 0; k < 4; k++) {
        const double2 q = project(R, t, cam, oc[k].x, oc[k].y, oc[k].z);
        const float dx = __fsub_rn(pu[k], (float)q.x), dy = __fsub_rn(pv[k], (float)q.y);
        if (!(sqrt((double)dx * dx + (double)dy * dy) < kGate2D)) return false;
    }
    return bb_area(a.ext + 3 * obj, R, t, (float)cam[0], (float)cam[1], (float)cam[2], (float)cam[3], a.W, a.H) >= kMinArea;
}

// grid (kHyp / kSampleWarps, B), one warp per hypothesis: lane i runs attempt base + i, a ballot keeps the lowest accepted attempt
// of each group of 32, so the result is the sequential loop's first accepted attempt.  exhausted[b] must be zero on entry.
__global__ void __launch_bounds__(kSampleWarps * 32)
k_sample2d(const Args a, int* __restrict__ exhausted)
{
    __shared__ int objs[kMaxC];
    __shared__ int nobj;
    const int b = blockIdx.y, lane = threadIdx.x & 31, h = blockIdx.x * kSampleWarps + (threadIdx.x >> 5);
    const int* counts = a.counts + (size_t)b * a.C;
    if (threadIdx.x == 0) {
        int n = 0;
        for (int c = 1; c < a.C; c++)
            if (counts[c] > kMinArea) objs[n++] = c;
        nobj = n;
    }
    __syncthreads();
    const float* m = a.meta + (size_t)b * a.num_meta;
    const double cam[4] = {m[0], m[4], m[2], m[5]};
    const uint64_t key = a.keys[b];
    double R[9], t[3];
    int obj = 0, pix[4], base = 0, win = -1;
    if (nobj > 0)
        for (; base < kMaxAttempts; base += 32) {
            const unsigned ok = __ballot_sync(0xffffffffu, attempt2d(a, b, objs, nobj, cam, key, h, base + lane, R, t, obj, pix));
            if (ok) { win = __ffs(ok) - 1; break; }
        }
    const bool found = win >= 0;
    if (lane == (found ? win : 0)) {
        Hyp& out = a.hyps[(size_t)b * kHyp + h];
        for (int k = 0; k < 9; k++) out.R[k] = found ? R[k] : 0.0;
        for (int k = 0; k < 3; k++) out.t[k] = found ? t[k] : 0.0;
        out.obj = found ? obj : 0;
        out.attempts = nobj == 0 ? 0 : found ? base + win + 1 : kMaxAttempts;
        if (a.trace_hyp) {
            int32_t* tr = a.trace_hyp + ((size_t)b * kHyp + h) * kTraceHyp2D;
            tr[0] = out.obj; tr[1] = out.attempts;
            for (int k = 0; k < 4; k++) tr[2 + k] = found ? pix[k] : -1;
            for (int r = 0; r < kRounds; r++) tr[6 + r] = -1;
        }
    }
    const int n_ex = __syncthreads_count(lane == 0 && nobj > 0 && !found);
    if (threadIdx.x == 0 && n_ex) atomicAdd(exhausted + b, n_ex);
}

// ------------------------------------------------------------------------------------------------- preemptive loop
struct RShared {
    int id[kHyp], cnt[kHyp], nid[kHyp], ncnt[kHyp];
    int n, T;
    unsigned mask[kWarps][kWords];
    int pref[kWarps][kWords];
    int fsel[kMaxInl];
    double R0[9], t0[3];           // survivor's pose at its last count
    double red[kWarps];
    double energy;
    // Nelder-Mead
    double x[7][6], f[7], xc[6], xr[6], xt[6], lb[6], ub[6], fr;
    int ord[7], evals, flag;
};
static_assert(sizeof(float) * 6 * kMaxInl <= sizeof(unsigned) * kWarps * kWords * 2, "final pairs reuse the mask storage");

// warp: inlier masks of (R, t) over the T taken pixels, exclusive popcount prefix per word; returns the inlier count
template <class Gate>
__device__ int warp_masks(RShared& s, int w, const double* R, const double* t, const float* teye, const float* tobj, int T, const Gate& gate)
{
    const int lane = threadIdx.x & 31, nw = (T + 31) / 32;
    int total = 0;
    for (int k = 0; k < nw; k++) {
        const int i = 32 * k + lane;
        bool in = false;
        if (i < T)
            in = gate(R, t, make_float3(teye[3 * i], teye[3 * i + 1], teye[3 * i + 2]),
                      make_float3(tobj[3 * i], tobj[3 * i + 1], tobj[3 * i + 2]));
        const unsigned bm = __ballot_sync(0xffffffffu, in);
        if (lane == 0) { s.mask[w][k] = bm; s.pref[w][k] = total; }
        total += __popc(bm);
    }
    __syncwarp();
    return total;
}

// the taken-pixel slot of the inlier of rank q (masks of warp w)
__device__ __forceinline__ int inlier_slot(const RShared& s, int w, int nw, int q)
{
    int lo = 0, hi = nw - 1;
    while (lo < hi) {            // last word with pref <= q
        const int mid = (lo + hi + 1) >> 1;
        if (s.pref[w][mid] <= q) lo = mid; else hi = mid - 1;
    }
    unsigned bm = s.mask[w][lo];
    for (int r = q - s.pref[w][lo]; r > 0; r--) bm &= bm - 1u;
    return 32 * lo + __ffs(bm) - 1;
}

// block: energy of optEnergy3D (:1464-1507) at the pose vector x: rotation rounded to float, mean distance over the m pairs
// (pairs in shared memory, obj then eye, 6 floats each); fixed-order double sum
__device__ double block_energy(RShared& s, const double* x, const float* pairs, int m)
{
    double Rd[9];
    rodrigues_exp(x, Rd);
    float Rf[9];
    for (int k = 0; k < 9; k++) Rf[k] = (float)Rd[k];
    double acc = 0.0;
    for (int j = threadIdx.x; j < m; j += kThreads) {
        const float* p = pairs + 6 * j;
        float q[3];
        for (int i = 0; i < 3; i++) {
            const float r = (float)((double)Rf[3 * i] * p[0] + (double)Rf[3 * i + 1] * p[1] + (double)Rf[3 * i + 2] * p[2]);
            q[i] = (float)((double)r + x[3 + i]);
        }
        const double dx = (double)q[0] - p[3], dy = (double)q[1] - p[4], dz = (double)q[2] - p[5];
        acc += sqrt(dx * dx + dy * dy + dz * dz);
    }
    acc = warp_sum(acc);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s.red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double sum = 0.0;
        for (int k = 0; k < kWarps; k++) sum += s.red[k];
        s.energy = (double)__fdiv_rn((float)sum, (float)m);
    }
    __syncthreads();
    return s.energy;
}

__device__ void nm_clamp(const RShared& s, double* x)
{
    for (int i = 0; i < 6; i++) x[i] = fmin(fmax(x[i], s.lb[i]), s.ub[i]);
}

// bounded Nelder-Mead (DESIGN §13): simplex x0 + half the bound radius along each axis, reflection 1, expansion 2, contractions
// and shrink 1/2, trial points clamped to the box, kNMEvals evaluations in all; s.x[best] / s.f[best] on return (best = s.ord[0])
__device__ void nelder_mead(RShared& s, const double* x0, const float* pairs, int m)
{
    const int t = threadIdx.x;
    const double range[6] = {10.0 * 3.1415926 / 180.0, 10.0 * 3.1415926 / 180.0, 10.0 * 3.1415926 / 180.0, 0.1, 0.1, 0.5};
    if (t == 0) {
        for (int i = 0; i < 6; i++) { s.lb[i] = x0[i] - range[i]; s.ub[i] = x0[i] + range[i]; }
        for (int v = 0; v < 7; v++) {
            for (int i = 0; i < 6; i++) s.x[v][i] = x0[i];
            if (v) s.x[v][v - 1] += 0.5 * range[v - 1];
            s.ord[v] = v;
        }
    }
    __syncthreads();
    for (int v = 0; v < 7; v++) {
        const double e = block_energy(s, s.x[v], pairs, m);
        if (t == 0) s.f[v] = e;
    }
    int evals = 7;
    while (evals < kNMEvals) {
        if (t == 0) {
            for (int i = 1; i < 7; i++)          // stable insertion sort of the vertices by energy
                for (int j = i; j > 0 && s.f[s.ord[j]] < s.f[s.ord[j - 1]]; j--) { const int q = s.ord[j]; s.ord[j] = s.ord[j - 1]; s.ord[j - 1] = q; }
            const int wv = s.ord[6];
            for (int i = 0; i < 6; i++) {
                double c = 0.0;
                for (int v = 0; v < 6; v++) c += s.x[s.ord[v]][i];
                s.xc[i] = c / 6.0;
                s.xr[i] = s.xc[i] + (s.xc[i] - s.x[wv][i]);
            }
            nm_clamp(s, s.xr);
        }
        __syncthreads();
        const double fr = block_energy(s, s.xr, pairs, m);
        evals++;
        if (t == 0) {
            const int wv = s.ord[6];
            s.fr = fr;
            if (fr < s.f[s.ord[0]]) {
                s.flag = 1;
                for (int i = 0; i < 6; i++) s.xt[i] = s.xc[i] + 2.0 * (s.xc[i] - s.x[wv][i]);
            } else if (fr < s.f[s.ord[5]]) {
                s.flag = 0;
            } else if (fr < s.f[wv]) {
                s.flag = 2;
                for (int i = 0; i < 6; i++) s.xt[i] = s.xc[i] + 0.5 * (s.xr[i] - s.xc[i]);
            } else {
                s.flag = 3;
                for (int i = 0; i < 6; i++) s.xt[i] = s.xc[i] + 0.5 * (s.x[wv][i] - s.xc[i]);
            }
            nm_clamp(s, s.xt);
            if (s.flag == 0) {
                for (int i = 0; i < 6; i++) s.x[wv][i] = s.xr[i];
                s.f[wv] = fr;
            }
        }
        __syncthreads();
        const int flag = s.flag;
        if (flag == 0) continue;
        if (evals >= kNMEvals) {
            if (flag == 1 && t == 0) {       // no budget for the expansion: keep the reflection
                const int wv = s.ord[6];
                for (int i = 0; i < 6; i++) s.x[wv][i] = s.xr[i];
                s.f[wv] = s.fr;
            }
            __syncthreads();
            break;
        }
        const double ft = block_energy(s, s.xt, pairs, m);
        evals++;
        if (t == 0) {
            const int wv = s.ord[6];
            const bool accept = flag == 1 || (flag == 2 ? ft <= s.fr : ft < s.f[wv]);
            s.flag = accept ? 0 : 4;
            if (flag == 1) {
                const bool exp = ft < s.fr;
                for (int i = 0; i < 6; i++) s.x[wv][i] = exp ? s.xt[i] : s.xr[i];
                s.f[wv] = exp ? ft : s.fr;
            } else if (accept) {
                for (int i = 0; i < 6; i++) s.x[wv][i] = s.xt[i];
                s.f[wv] = ft;
            }
        }
        __syncthreads();
        if (s.flag == 4) {                  // shrink towards the best vertex
            for (int k = 1; k < 7 && evals < kNMEvals; k++) {
                if (t == 0) {
                    const int v = s.ord[k], bv = s.ord[0];
                    for (int i = 0; i < 6; i++) s.x[v][i] = s.x[bv][i] + 0.5 * (s.x[v][i] - s.x[bv][i]);
                }
                __syncthreads();
                const double e = block_energy(s, s.x[s.ord[k]], pairs, m);
                evals++;
                if (t == 0) s.f[s.ord[k]] = e;
            }
            __syncthreads();
        }
    }
    if (t == 0)
        for (int i = 1; i < 7; i++)
            for (int j = i; j > 0 && s.f[s.ord[j]] < s.f[s.ord[j - 1]]; j--) { const int q = s.ord[j]; s.ord[j] = s.ord[j - 1]; s.ord[j - 1] = q; }
    __syncthreads();
}

// k2D: the colour-only estimator (estimatePose2D): taken pixels hold (x, y, 0) instead of camera points, the inlier test is the
// 10 px reprojection gate, and there is no refit and no Nelder-Mead (the reference's updateHyp3D returns at once on a 2-D
// hypothesis, and optEnergy2D divides by its empty 3-D inlier list, DESIGN §13): the survivor keeps its P3P pose
template <bool k2D>
__global__ void __launch_bounds__(kThreads, 1)
k_ransac(const Args a)
{
    __shared__ RShared s;
    const int c = blockIdx.x, b = blockIdx.y, t = threadIdx.x, w = t >> 5, lane = t & 31;
    const int HW = a.H * a.W;
    const int N = a.counts[(size_t)b * a.C + c];
    float* pose = a.poses + ((size_t)b * a.C + c) * 12;
    float* info = a.info + ((size_t)b * a.C + c) * kInfo;
    int32_t* trr = a.trace_round ? a.trace_round + ((size_t)b * a.C + c) * kRounds * kTraceRound : nullptr;
    const Hyp* hyps = a.hyps + (size_t)b * kHyp;
    // hypotheses of this class, in hypothesis order
    const bool mine = c > 0 && N > kMinArea && hyps[t].obj == c;
    const unsigned bm = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) s.nid[w] = __popc(bm);
    __syncthreads();
    int before = 0, n0 = 0;
    for (int k = 0; k < kWarps; k++) { before += k < w ? s.nid[k] : 0; n0 += s.nid[k]; }
    __syncthreads();
    if (mine) s.id[before + __popc(bm & ((1u << lane) - 1u))] = t;
    if (t < 12) pose[t] = 0.f;
    if (trr)
        for (int i = t; i < kRounds * kTraceRound; i += kThreads) trr[i] = 0;
    if (n0 == 0) {
        if (t < kInfo) info[t] = t == 0 ? (float)(c > 0 ? N : 0) : (t == 3 || t == 5) ? -1.f : (t == 4 && c > 0) ? (float)a.exhausted[b] : 0.f;
        return;
    }
    if (t == 0) s.n = n0;
    __syncthreads();
    const float* m = a.meta + (size_t)b * a.num_meta;
    const float fx = m[0], px = m[2], fy = m[4], py = m[5];
    const uint64_t key = a.keys[b];
    const int* L = a.list + (size_t)b * HW + a.start[(size_t)b * a.C + c];
    const size_t slot = (size_t)b * (a.C - 1) + (c - 1);     // class 0 never has a slot
    int* taken = a.taken + slot * kMaxTaken;
    float* teye = a.teye + slot * kMaxTaken * 3;
    float* tobj = a.tobj + slot * kMaxTaken * 3;
    Hyp* H = a.hyps + (size_t)b * kHyp;
    const std::conditional_t<k2D, Gate2D, Gate3D> gate(fx, fy, px, py);

    for (int r = 0; r < kRounds; r++) {
        const int maxPixels = kBatch * (r + 1);
        // ---- the round's pixel subset (countInliers3D's stepping rule), warp 0
        if (w == 0) {
            const float p = __fdiv_rn((float)maxPixels, (float)N);
            const bool all = !(p < 1.f);
            const double lq = all ? 0.0 : log1p(-(double)p);
            int pos = 0, T = 0;
            uint64_t k = 0;
            unsigned hash = 0;
            while (pos < N && T < kMaxTaken) {
                int st = 1;
                if (!all) {
                    uint32_t wd[4];
                    philox4x32_10(key, ctr_sub(c, r, k + lane), wd);
                    const double u = (double)(((((uint64_t)wd[0] << 32) | wd[1]) >> 11) + 1) * 0x1p-53;
                    const double g = floor(log(u) / lq);
                    st = g < 1.0 ? 1 : (g > (double)N ? N : (int)g);
                }
                int incl = st;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                const int cand = pos + incl - st;
                const int entry = cand < N ? __ldg(L + cand) : (int)kHole;
                const unsigned bad = __ballot_sync(0xffffffffu, cand >= N || (entry & (int)kHole));
                const int f = min(bad ? __ffs(bad) - 1 : 32, kMaxTaken - T);
                if (lane < f) { taken[T + lane] = entry; hash += (unsigned)entry; }
                T += f;
                k += f;
                if (T >= kMaxTaken) break;
                if (!bad) { pos = __shfl_sync(0xffffffffu, cand + st, 31); continue; }
                pos = __shfl_sync(0xffffffffu, cand, f);
                if (pos >= N) break;
                for (pos += 1; pos < N; pos += 32) {        // holes advance by one and take no draw
                    const int q = pos + lane;
                    const unsigned ok = __ballot_sync(0xffffffffu, q < N && !(__ldg(L + q) & (int)kHole));
                    if (ok) { pos += __ffs(ok) - 1; break; }
                }
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) hash += __shfl_xor_sync(0xffffffffu, hash, o);
            if (lane == 0) {
                s.T = T;
                if (trr) { trr[r * kTraceRound] = T; trr[r * kTraceRound + 1] = (int)hash; }
            }
        }
        __syncthreads();
        const int T = s.T;
        for (int i = t; i < T; i += kThreads) {
            const int idx = taken[i];
            float3 e;
            if constexpr (k2D)
                e = make_float3((float)(idx % a.W), (float)(idx / a.W), 0.f);
            else
                e = eye_at(a.depth + (size_t)b * HW, a.W, fx, fy, px, py, a.factor, idx);
            const float3 o = mode_at(a, b, c, idx);
            teye[3 * i] = e.x; teye[3 * i + 1] = e.y; teye[3 * i + 2] = e.z;
            tobj[3 * i] = o.x; tobj[3 * i + 1] = o.y; tobj[3 * i + 2] = o.z;
        }
        __syncthreads();
        // ---- inlier counts, one warp per hypothesis
        const int n = s.n;
        for (int k = w; k < n; k += kWarps) {
            const Hyp& hy = H[s.id[k]];
            const int cntk = warp_masks(s, w, hy.R, hy.t, teye, tobj, T, gate);
            if (lane == 0) {
                s.cnt[k] = cntk;
                if (a.trace_hyp)
                    a.trace_hyp[((size_t)b * kHyp + s.id[k]) * (k2D ? kTraceHyp2D : kTraceHyp) + (k2D ? 6 : 5) + r] = cntk;
            }
        }
        __syncthreads();
        // ---- sort by inliers (descending, ties by hypothesis index), keep the first n / 2
        const int keep = n > 1 ? n / 2 : n;
        if (t < n) {
            const int ci = s.cnt[t], ii = s.id[t];
            int rank = 0;
            for (int j = 0; j < n; j++) rank += s.cnt[j] > ci || (s.cnt[j] == ci && s.id[j] < ii);
            if (rank < keep) { s.nid[rank] = ii; s.ncnt[rank] = ci; }
        }
        __syncthreads();
        if (t < keep) { s.id[t] = s.nid[t]; s.cnt[t] = s.ncnt[t]; }
        if (t == 0) {
            s.n = keep;
            if (trr) { trr[r * kTraceRound + 2] = s.nid[0]; trr[r * kTraceRound + 3] = s.ncnt[0]; }
        }
        __syncthreads();
        // ---- refine every hypothesis still in the queue (updateHyp3D): Kabsch on <= 1000 inliers; none in 2-D
        for (int k = w; !k2D && k < keep; k += kWarps) {
            const int h = s.id[k], ninl = s.cnt[k];
            Hyp& hy = H[h];
            if (r == kRounds - 1 && lane == 0) {          // keep = 1 here: the pose of the survivor's last count
                for (int i = 0; i < 9; i++) s.R0[i] = hy.R[i];
                for (int i = 0; i < 3; i++) s.t0[i] = hy.t[i];
            }
            if (ninl < 4) continue;
            double Rc[9], tc[3];
            for (int i = 0; i < 9; i++) Rc[i] = hy.R[i];
            for (int i = 0; i < 3; i++) tc[i] = hy.t[i];
            warp_masks(s, w, Rc, tc, teye, tobj, T, gate);
            const int nw = (T + 31) / 32, mm = ninl >= kMaxInl ? kMaxInl : ninl;
            double sa[6] = {0, 0, 0, 0, 0, 0};
            for (int j = lane; j < mm; j += 32) {
                int q = j;
                if (ninl >= kMaxInl) { uint32_t wd[4]; philox4x32_10(key, ctr_fil(h, r, j), wd); q = uniform_int(wd[0], ninl); }
                const int i = inlier_slot(s, w, nw, q);
                for (int d = 0; d < 3; d++) { sa[d] += tobj[3 * i + d]; sa[3 + d] += teye[3 * i + d]; }
            }
            double cA[3], cB[3];
            for (int d = 0; d < 3; d++) { cA[d] = warp_sum(sa[d]) * (1.0 / mm); cB[d] = warp_sum(sa[3 + d]) * (1.0 / mm); }
            double cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            for (int j = lane; j < mm; j += 32) {
                int q = j;
                if (ninl >= kMaxInl) { uint32_t wd[4]; philox4x32_10(key, ctr_fil(h, r, j), wd); q = uniform_int(wd[0], ninl); }
                const int i = inlier_slot(s, w, nw, q);
                const double pa[3] = {tobj[3 * i] - cA[0], tobj[3 * i + 1] - cA[1], tobj[3 * i + 2] - cA[2]};
                const double pb[3] = {teye[3 * i] - cB[0], teye[3 * i + 1] - cB[1], teye[3 * i + 2] - cB[2]};
                for (int x = 0; x < 3; x++)
                    for (int y = 0; y < 3; y++) cov[3 * x + y] += pa[x] * pb[y];
            }
            for (int x = 0; x < 9; x++) cov[x] = warp_sum(cov[x]);
            if (lane == 0) {
                double Rn[9], tn[3];
                if (kabsch(cov, cA, cB, Rn, tn)) {
                    for (int i = 0; i < 9; i++) hy.R[i] = Rn[i];
                    for (int i = 0; i < 3; i++) hy.t[i] = tn[i];
                }
            }
            __syncwarp();
        }
        __syncthreads();
    }

    // ---- the survivor: Nelder-Mead over a fresh filtered set of its last inliers
    const int h = s.id[0], inl = s.cnt[0];
    const Hyp& hy = H[h];
    double Rout[9], tout[3];
    for (int i = 0; i < 9; i++) Rout[i] = hy.R[i];
    for (int i = 0; i < 3; i++) tout[i] = hy.t[i];
    double energy = -1.0;
    if (!k2D && inl > kMinFinal) {
        const int T = s.T, nw = (T + 31) / 32;
        if (w == 0) warp_masks(s, 0, s.R0, s.t0, teye, tobj, T, gate);
        __syncthreads();
        const int mm = inl >= kMaxInl ? kMaxInl : inl;
        for (int j = t; j < mm; j += kThreads) {
            int q = j;
            if (inl >= kMaxInl) {         // the last refinement's filtered list, filtered once more (:1942)
                uint32_t wd[4];
                philox4x32_10(key, ctr_fil(h, kRounds, j), wd);
                const int i1 = uniform_int(wd[0], kMaxInl);
                philox4x32_10(key, ctr_fil(h, kRounds - 1, i1), wd);
                q = uniform_int(wd[0], inl);
            }
            s.fsel[j] = inlier_slot(s, 0, nw, q);
        }
        __syncthreads();
        float* pairs = reinterpret_cast<float*>(&s.mask[0][0]);
        for (int j = t; j < mm; j += kThreads) {
            const int i = s.fsel[j];
            for (int d = 0; d < 3; d++) { pairs[6 * j + d] = tobj[3 * i + d]; pairs[6 * j + 3 + d] = teye[3 * i + d]; }
        }
        __syncthreads();
        double x0[6];
        rodrigues_log(Rout, x0);
        for (int i = 0; i < 3; i++) x0[3 + i] = tout[i];
        nelder_mead(s, x0, pairs, mm);
        const int bv = s.ord[0];
        rodrigues_exp(s.x[bv], Rout);
        for (int i = 0; i < 3; i++) tout[i] = s.x[bv][3 + i];
        energy = s.f[bv];
    }
    if (t == 0) {
        for (int i = 0; i < 3; i++) {
            for (int j = 0; j < 3; j++) pose[4 * i + j] = (float)Rout[3 * i + j];
            pose[4 * i + 3] = (float)tout[i];
        }
        info[0] = (float)N;
        info[1] = (float)n0;
        info[2] = (float)inl;
        info[3] = (float)energy;
        info[4] = (float)a.exhausted[b];
        info[5] = (float)h;
    }
}

// ------------------------------------------------------------------------------------------------- detection records
// transforms3d's quat2mat on float32 values (numpy float32 scalars in test.py's _get_bb2D)
__device__ void quat2mat_f(const float* q, float* R)
{
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    const float Nq = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w, w), __fmul_rn(x, x)), __fmul_rn(y, y)), __fmul_rn(z, z));
    if (Nq < 2.220446049250313e-16f * 4.f) {
        for (int k = 0; k < 9; k++) R[k] = (k % 4 == 0) ? 1.f : 0.f;
        return;
    }
    const float s = __fdiv_rn(2.f, Nq);
    const float X = __fmul_rn(x, s), Y = __fmul_rn(y, s), Z = __fmul_rn(z, s);
    const float wX = __fmul_rn(w, X), wY = __fmul_rn(w, Y), wZ = __fmul_rn(w, Z);
    const float xX = __fmul_rn(x, X), xY = __fmul_rn(x, Y), xZ = __fmul_rn(x, Z);
    const float yY = __fmul_rn(y, Y), yZ = __fmul_rn(y, Z), zZ = __fmul_rn(z, Z);
    R[0] = __fsub_rn(1.f, __fadd_rn(yY, zZ)); R[1] = __fsub_rn(xY, wZ);                 R[2] = __fadd_rn(xZ, wY);
    R[3] = __fadd_rn(xY, wZ);                 R[4] = __fsub_rn(1.f, __fadd_rn(xX, zZ)); R[5] = __fsub_rn(yZ, wX);
    R[6] = __fsub_rn(xZ, wY);                 R[7] = __fadd_rn(yZ, wX);                 R[8] = __fsub_rn(1.f, __fadd_rn(xX, yY));
}

// the records of lib/fcn/test.py:1383-1399 for every image of the batch: for each class j ascending with t_z > 0,
// rois = (image, j, _get_bb2D(extent, pose, K) * im_scale) (test.py:1115-1148, K = the unscaled intrinsics), poses = (mat2quat(R), t);
// rows of all images in (image, class) order, zero rows after them, the row count in *num.  One CTA.
__global__ void __launch_bounds__(kRecThreads)
k_records(const float* __restrict__ poses, const float* __restrict__ ext, const float* __restrict__ meta, int num_meta, int B, int C,
          int batch_offset, float im_scale, float* __restrict__ rois, float* __restrict__ oposes, int32_t* __restrict__ num)
{
    __shared__ int wsum[kRecThreads / 32];
    __shared__ int base;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5, n = B * (C - 1);
    if (t == 0) base = 0;
    __syncthreads();
    for (int c0 = 0; c0 < n; c0 += kRecThreads) {
        const int i = c0 + t, b = i / (C - 1), c = i % (C - 1) + 1;
        const float* P = poses + ((size_t)b * C + c) * 12;
        const bool flag = i < n && P[11] > 0.f;
        const unsigned bm = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) wsum[w] = __popc(bm);
        __syncthreads();
        int before = base, total = 0;
        for (int k = 0; k < kRecThreads / 32; k++) { before += k < w ? wsum[k] : 0; total += wsum[k]; }
        if (flag) {
            const int r = before + __popc(bm & ((1u << lane) - 1u));
            float q[4], R[9];
            mat2quat_d(P, q);
            quat2mat_f(q, R);
            const float* m = meta + (size_t)b * num_meta;
            const double fx = (double)m[0] / im_scale, px = (double)m[2] / im_scale, fy = (double)m[4] / im_scale,
                         py = (double)m[5] / im_scale;
            const float* e = ext + 3 * c;
            const float hx = __fmul_rn(e[0], 0.5f), hy = __fmul_rn(e[1], 0.5f), hz = __fmul_rn(e[2], 0.5f);
            double x0 = INFINITY, x1 = -INFINITY, y0 = INFINITY, y1 = -INFINITY;
            for (int k = 0; k < 8; k++) {       // the corner order of _get_bb2D does not change the extremes
                const float X = (k & 1) ? -hx : hx, Y = (k & 2) ? -hy : hy, Z = (k & 4) ? -hz : hz;
                float Pc[3];
                for (int j = 0; j < 3; j++)
                    Pc[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[3 * j], X), __fmul_rn(R[3 * j + 1], Y)), __fmul_rn(R[3 * j + 2], Z)),
                                      P[4 * j + 3]);
                const double u = (fx * Pc[0] + px * Pc[2]) / (double)Pc[2], v = (fy * Pc[1] + py * Pc[2]) / (double)Pc[2];
                x0 = fmin(x0, u); x1 = fmax(x1, u); y0 = fmin(y0, v); y1 = fmax(y1, v);
            }
            float* ro = rois + (size_t)r * 6;
            ro[0] = (float)(b + batch_offset); ro[1] = (float)c;
            ro[2] = __fmul_rn((float)x0, im_scale); ro[3] = __fmul_rn((float)y0, im_scale);
            ro[4] = __fmul_rn((float)x1, im_scale); ro[5] = __fmul_rn((float)y1, im_scale);
            float* po = oposes + (size_t)r * 7;
            for (int k = 0; k < 4; k++) po[k] = q[k];
            po[4] = P[3]; po[5] = P[7]; po[6] = P[11];
        }
        __syncthreads();
        if (t == 0) base += total;
        __syncthreads();
    }
    for (int r = base + t; r < n; r += kRecThreads) {
        for (int k = 0; k < 6; k++) rois[(size_t)r * 6 + k] = 0.f;
        for (int k = 0; k < 7; k++) oposes[(size_t)r * 7 + k] = 0.f;
    }
    if (t == 0) *num = base;
}

struct Layout {
    size_t counts, start, exhausted, list, hyps, taken, teye, tobj, total;
};

Layout layout(int B, int H, int W, int C)
{
    Layout l;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align_up(o + bytes, 256); return at; };
    const size_t slots = (size_t)B * (C - 1);
    l.counts = take((size_t)B * C * sizeof(int));
    l.start = take((size_t)B * C * sizeof(int));
    l.exhausted = take((size_t)B * sizeof(int));
    l.list = take((size_t)B * H * W * sizeof(int));
    l.hyps = take((size_t)B * kHyp * sizeof(Hyp));
    l.taken = take(slots * kMaxTaken * sizeof(int));
    l.teye = take(slots * kMaxTaken * 3 * sizeof(float));
    l.tobj = take(slots * kMaxTaken * 3 * sizeof(float));
    l.total = o;
    return l;
}

}  // namespace coordpose
}  // namespace pcnn

using namespace pcnn;
using namespace pcnn::coordpose;

extern "C" int pcnn_coord_pose3d_workspace_bytes(int B, int H, int W, int C, size_t* bytes)
{
    PCNN_REQUIRE(bytes, "coord_pose3d: bytes is NULL");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "coord_pose3d: bad shape B = %d, H = %d, W = %d", B, H, W);
    PCNN_REQUIRE(C >= 2 && C <= kMaxC, "coord_pose3d: C = %d outside [2, %d]", C, kMaxC);
    PCNN_REQUIRE((size_t)H * W <= (size_t)(INT_MAX / 64), "coord_pose3d: image too large");
    *bytes = layout(B, H, W, C).total;
    return PCNN_OK;
}

extern "C" int pcnn_coord_pose3d_fwd(const int32_t* label, const float* vertex, const float* lowres, const float* bias_vertex,
                                     const float* depth, const float* meta, int num_meta, const float* extents, const uint64_t* keys,
                                     int B, int H, int W, int C, float depth_factor, float* poses, float* info, int32_t* trace_hyp,
                                     int32_t* trace_round, void* workspace, size_t workspace_bytes, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    PCNN_REQUIRE(label && depth && meta && extents && keys && poses && info && workspace, "coord_pose3d: NULL required pointer");
    PCNN_REQUIRE(vertex || (lowres && bias_vertex), "coord_pose3d: need the dense vertex tensor or lowres + bias_vertex");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "coord_pose3d: bad shape B = %d, H = %d, W = %d", B, H, W);
    PCNN_REQUIRE(C >= 2 && C <= kMaxC, "coord_pose3d: C = %d outside [2, %d]", C, kMaxC);
    PCNN_REQUIRE(vertex || (H % 8 == 0 && W % 8 == 0), "coord_pose3d: the lowres source needs H, W multiples of 8 (got %d x %d)", H, W);
    PCNN_REQUIRE((size_t)H * W <= (size_t)(INT_MAX / 64), "coord_pose3d: image too large");
    PCNN_REQUIRE(num_meta >= 6, "coord_pose3d: num_meta = %d < 6", num_meta);
    PCNN_REQUIRE(depth_factor > 0.f, "coord_pose3d: depth_factor must be > 0");
    const Layout l = layout(B, H, W, C);
    PCNN_REQUIRE(workspace_bytes >= l.total, "coord_pose3d: workspace %zu B < %zu B", workspace_bytes, l.total);
    char* ws = (char*)workspace;
    Args a{label, depth, vertex, vertex ? nullptr : lowres, vertex ? nullptr : bias_vertex, meta, extents, keys, num_meta, B, H, W, C,
           depth_factor, (const int*)(ws + l.counts), (const int*)(ws + l.start), (const int*)(ws + l.list),
           (const int*)(ws + l.exhausted), (Hyp*)(ws + l.hyps), (int*)(ws + l.taken), (float*)(ws + l.teye), (float*)(ws + l.tobj),
           poses, info, trace_hyp, trace_round};
    k_lists<true><<<B, kListThreads, 0, stream>>>(label, depth, H, W, C, (int*)(ws + l.counts), (int*)(ws + l.start), (int*)(ws + l.list));
    int rc = check_launch("coord_pose3d: pixel lists");
    if (rc) return rc;
    k_sample<<<B, kHyp, 0, stream>>>(a, (int*)(ws + l.exhausted));
    rc = check_launch("coord_pose3d: hypotheses");
    if (rc) return rc;
    k_ransac<false><<<dim3(C, B), kThreads, 0, stream>>>(a);
    return check_launch("coord_pose3d: preemptive RANSAC");
}

extern "C" int pcnn_coord_pose2d_workspace_bytes(int B, int H, int W, int C, size_t* bytes)
{
    PCNN_REQUIRE(bytes, "coord_pose2d: bytes is NULL");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "coord_pose2d: bad shape B = %d, H = %d, W = %d", B, H, W);
    PCNN_REQUIRE(C >= 2 && C <= kMaxC, "coord_pose2d: C = %d outside [2, %d]", C, kMaxC);
    PCNN_REQUIRE((size_t)H * W <= (size_t)(INT_MAX / 64), "coord_pose2d: image too large");
    *bytes = layout(B, H, W, C).total;
    return PCNN_OK;
}

extern "C" int pcnn_coord_pose2d_fwd(const int32_t* label, const float* vertex, const float* lowres, const float* bias_vertex,
                                     const float* meta, int num_meta, const float* extents, const uint64_t* keys, int B, int H, int W,
                                     int C, float* poses, float* info, int32_t* trace_hyp, int32_t* trace_round, void* workspace,
                                     size_t workspace_bytes, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    PCNN_REQUIRE(label && meta && extents && keys && poses && info && workspace, "coord_pose2d: NULL required pointer");
    PCNN_REQUIRE(vertex || (lowres && bias_vertex), "coord_pose2d: need the dense vertex tensor or lowres + bias_vertex");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1, "coord_pose2d: bad shape B = %d, H = %d, W = %d", B, H, W);
    PCNN_REQUIRE(C >= 2 && C <= kMaxC, "coord_pose2d: C = %d outside [2, %d]", C, kMaxC);
    PCNN_REQUIRE(vertex || (H % 8 == 0 && W % 8 == 0), "coord_pose2d: the lowres source needs H, W multiples of 8 (got %d x %d)", H, W);
    PCNN_REQUIRE((size_t)H * W <= (size_t)(INT_MAX / 64), "coord_pose2d: image too large");
    PCNN_REQUIRE(num_meta >= 6, "coord_pose2d: num_meta = %d < 6", num_meta);
    const Layout l = layout(B, H, W, C);
    PCNN_REQUIRE(workspace_bytes >= l.total, "coord_pose2d: workspace %zu B < %zu B", workspace_bytes, l.total);
    char* ws = (char*)workspace;
    Args a{label, nullptr, vertex, vertex ? nullptr : lowres, vertex ? nullptr : bias_vertex, meta, extents, keys, num_meta, B, H, W, C,
           1.f, (const int*)(ws + l.counts), (const int*)(ws + l.start), (const int*)(ws + l.list),
           (const int*)(ws + l.exhausted), (Hyp*)(ws + l.hyps), (int*)(ws + l.taken), (float*)(ws + l.teye), (float*)(ws + l.tobj),
           poses, info, trace_hyp, trace_round};
    k_lists<false><<<B, kListThreads, 0, stream>>>(label, nullptr, H, W, C, (int*)(ws + l.counts), (int*)(ws + l.start), (int*)(ws + l.list));
    int rc = check_launch("coord_pose2d: pixel lists");
    if (rc) return rc;
    if (cudaMemsetAsync(ws + l.exhausted, 0, (size_t)B * sizeof(int), stream) != cudaSuccess) return check_launch("coord_pose2d: memset");
    k_sample2d<<<dim3(kHyp / kSampleWarps, B), kSampleWarps * 32, 0, stream>>>(a, (int*)(ws + l.exhausted));
    rc = check_launch("coord_pose2d: hypotheses");
    if (rc) return rc;
    k_ransac<true><<<dim3(C, B), kThreads, 0, stream>>>(a);
    return check_launch("coord_pose2d: preemptive RANSAC");
}

extern "C" int pcnn_coord_pose3d_records(const float* poses, const float* extents, const float* meta, int num_meta, int B, int C,
                                         int batch_offset, float im_scale, float* rois, float* out_poses, int32_t* num_rows, void* stream_)
{
    PCNN_REQUIRE(poses && extents && meta && rois && out_poses && num_rows, "coord_pose3d_records: NULL required pointer");
    PCNN_REQUIRE(B >= 1 && C >= 2 && C <= kMaxC, "coord_pose3d_records: bad shape B = %d, C = %d", B, C);
    PCNN_REQUIRE(num_meta >= 6, "coord_pose3d_records: num_meta = %d < 6", num_meta);
    PCNN_REQUIRE(im_scale > 0.f, "coord_pose3d_records: im_scale must be > 0");
    k_records<<<1, kRecThreads, 0, (cudaStream_t)stream_>>>(poses, extents, meta, num_meta, B, C, batch_offset, im_scale, rois, out_poses,
                                                     num_rows);
    return check_launch("coord_pose3d_records");
}
