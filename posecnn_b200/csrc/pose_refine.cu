// pose_refine.cu — depth-based pose refinement of the post-NMS detections (DESIGN.md §12), the device counterpart of the
// reference's Synthesizer::icp_python / solveICP (lib/synthesize/synthesize.cpp:2031-2395) on the model point table.
//
//   k_class_hist     [B, C] int32 class-pixel counts of the label map: warp-aggregated shared-memory histogram, one global
//                    atomic per (CTA, class)
//   k_pose_refine    one launch for the batch: a cluster of 8 CTAs per ROI row, CTA h = depth hypothesis h.  Every CTA runs
//                    stage 1 (depth re-centring) redundantly, then its Gauss-Newton iterations and its score with the P points
//                    strided over the block; before every association pass a shared-memory depth grid of the transformed
//                    points marks the self-occluded ones (the reference associates against a render); fp64 per-point terms and per-thread partial sums, fixed-order block reduction,
//                    one thread does the 6x6 LDLT and the SE3 exp; the score's window search runs in fp32.  Scores gather at cluster rank 0 through distributed shared memory.
// No host synchronisation: num_rows is read on the device, rows past it are written as zeros.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <limits.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace pcnn {

constexpr int kRefThreads = 256;
constexpr int kRefWarps = kRefThreads / 32;
constexpr int kRefHyp = 8;
constexpr int kRefMaxPoints = 4096;
constexpr int kRefSums = 27;             // 21 (upper triangle of A) + 6 (g)
constexpr int kRefMinInliers = 6;
constexpr int kHistThreads = 256;
// self-occlusion of the model (stands in for the reference's render): a grid of square cells over the projected bounding box of
// the points, side max(sqrt(8 bw bh / P), max(bw, bh) / 64, 1) pixels; a point is visible within 3 mm of its cell's nearest point
constexpr double kVisPointsPerCell = 8.0;
constexpr int kVisMaxSide = 64;
constexpr int kVisMaxCells = (kVisMaxSide + 1) * (kVisMaxSide + 1);
constexpr double kVisMargin = 0.003;

__constant__ double c_dz[kRefHyp] = {0.0, -0.02, -0.01, 0.01, 0.02, 0.03, 0.04, 0.05};

struct RefImage {
    const int32_t* label;    // image b, [H,W]
    const float* depth;      // image b, [H,W] raw
    int H, W, c;
    float fx, fy, px, py, factor, znear, zfar, max_error;
};

__device__ __forceinline__ bool live_vertex(const RefImage& im, int u, int v, float3& X)
{
    const size_t i = (size_t)v * im.W + u;
    if (__ldg(im.label + i) != im.c) return false;
    const float z = __ldg(im.depth + i) / im.factor;
    if (!(z > im.znear && z < im.zfar)) return false;
    X = make_float3((u - im.px) * z / im.fx, (v - im.py) * z / im.fy, z);
    return true;
}

__device__ __forceinline__ double3 transform_d(const double* R, const double* t, float3 mf)
{
    const double mx = mf.x, my = mf.y, mz = mf.z;
    return make_double3(R[0] * mx + R[1] * my + R[2] * mz + t[0], R[3] * mx + R[4] * my + R[5] * mz + t[1],
                        R[6] * mx + R[7] * my + R[8] * mz + t[2]);
}

__device__ __forceinline__ float3 transform(const float* R, const float* t, float3 m)
{
    return make_float3(R[0] * m.x + R[1] * m.y + R[2] * m.z + t[0], R[3] * m.x + R[4] * m.y + R[5] * m.z + t[1],
                       R[6] * m.x + R[7] * m.y + R[8] * m.z + t[2]);
}

// projective association of the transformed model point q; true for an inlier (X, n, e filled).  fp64: the normal equations of a nearly symmetric object are ill-conditioned (condition numbers
// of 1e6 occur), so the per-point terms and their sums are formed in double; the score search stays fp32
__device__ __forceinline__ bool live_vertex_d(const RefImage& im, int u, int v, double3& X)
{
    const size_t i = (size_t)v * im.W + u;
    if (__ldg(im.label + i) != im.c) return false;
    const double z = (double)__ldg(im.depth + i) / (double)im.factor;
    if (!(z > im.znear && z < im.zfar)) return false;
    X = make_double3((u - (double)im.px) * z / im.fx, (v - (double)im.py) * z / im.fy, z);
    return true;
}

struct VisGrid {
    double u0, v0, side;
    int gw;
};

__device__ __forceinline__ int vis_cell(const RefImage& im, const VisGrid& g, double3 q)
{
    const double fu = im.fx * q.x / q.z + im.px, fv = im.fy * q.y / q.z + im.py;
    return (int)((fv - g.v0) / g.side) * g.gw + (int)((fu - g.u0) / g.side);
}

__device__ bool associate_d(const RefImage& im, const VisGrid& g, const unsigned long long* zbuf, double3 q, double3& X, double3& n,
                            double& e)
{
    if (!(q.z > im.znear && q.z < im.zfar)) return false;
    if (!(q.z <= __longlong_as_double((long long)zbuf[vis_cell(im, g, q)]) + kVisMargin)) return false;   // occluded
    const double fu = im.fx * q.x / q.z + im.px + 0.5;
    const double fv = im.fy * q.y / q.z + im.py + 0.5;
    if (!(fu >= 3.0 && fu < (double)(im.W - 3) && fv >= 3.0 && fv < (double)(im.H - 3))) return false;   // 2 < u < W - 3
    const int u = (int)fu, v = (int)fv;
    double3 xl, xr, yu, yd;
    if (!live_vertex_d(im, u, v, X) || !live_vertex_d(im, u + 1, v, xr) || !live_vertex_d(im, u - 1, v, xl) ||
        !live_vertex_d(im, u, v + 1, yd) || !live_vertex_d(im, u, v - 1, yu))
        return false;
    const double ax = xr.x - xl.x, ay = xr.y - xl.y, az = xr.z - xl.z;
    const double bx = yd.x - yu.x, by = yd.y - yu.y, bz = yd.z - yu.z;
    n = make_double3(ay * bz - az * by, az * bx - ax * bz, ax * by - ay * bx);
    const double len = sqrt(n.x * n.x + n.y * n.y + n.z * n.z);
    if (!(len > 0.0)) return false;
    n = make_double3(n.x / len, n.y / len, n.z / len);
    if (n.x * X.x + n.y * X.y + n.z * X.z > 0.0) n = make_double3(-n.x, -n.y, -n.z);
    const double qn = sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    if (!(-(q.x * n.x + q.y * n.y + q.z * n.z) / qn >= 0.1)) return false;
    e = n.x * (X.x - q.x) + n.y * (X.y - q.y) + n.z * (X.z - q.z);
    return fabs(e) <= (double)im.max_error;
}

struct RefShared {
    double red[kRefWarps][kRefSums];
    int redc[kRefWarps];
    double sum[kRefSums];
    int count;
    double q[4], t[3];          // current pose (fp64)
    double Rd[9];               // its rotation matrix
    float R[9], tf[3];          // fp32 copy for the score search
    double q1[4], t1[3];        // stage 1 result
    int stop;
    double ext[kRefWarps][4];   // projected bounding box partials
    VisGrid grid;
    int ncells;
    // read by cluster rank 0 through distributed shared memory
    int score;
    int inliers;
    float pose[7];
};

// fixed-order block sum: per-thread fp64 partial sums -> xor butterfly per warp -> warps in index order
template <int N>
__device__ void block_sum(RefShared& s, const double (&v)[N], int cnt)
{
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
#pragma unroll
    for (int j = 0; j < N; j++) {
        double x = v[j];
#pragma unroll
        for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) s.red[w][j] = x;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s.redc[w] = cnt;
    __syncthreads();
    if (t < N) {
        double acc = 0.0;
        for (int k = 0; k < kRefWarps; k++) acc += s.red[k][t];
        s.sum[t] = acc;
    }
    if (t == N) {
        int acc = 0;
        for (int k = 0; k < kRefWarps; k++) acc += s.redc[k];
        s.count = acc;
    }
    __syncthreads();
}

__device__ void quat_mul(const double* a, const double* b, double* o)
{
    o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
    o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
    o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
    o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}

__device__ void quat_to_rot(const double* q, double* R)
{
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z);     R[2] = 2 * (x * z + w * y);
    R[3] = 2 * (x * y + w * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
    R[6] = 2 * (x * z - w * y);     R[7] = 2 * (y * z + w * x);     R[8] = 1 - 2 * (x * x + y * y);
}

__device__ void quat_normalize(double* q)
{
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    if (n == 0.0) { q[0] = 1.0; q[1] = q[2] = q[3] = 0.0; return; }
    for (int k = 0; k < 4; k++) q[k] /= n;
}

// thread 0: round the current pose to fp32 (the format of the outputs and of the trace, so that every step can be replayed from
// the trace exactly), then its rotation matrix (fp64 and fp32) and fp32 translation
__device__ void publish_pose(RefShared& s)
{
    for (int k = 0; k < 4; k++) s.q[k] = (double)(float)s.q[k];
    for (int k = 0; k < 3; k++) s.t[k] = (double)(float)s.t[k];
    double qn[4] = {s.q[0], s.q[1], s.q[2], s.q[3]};
    quat_normalize(qn);
    quat_to_rot(qn, s.Rd);
    for (int k = 0; k < 9; k++) s.R[k] = (float)s.Rd[k];
    for (int k = 0; k < 3; k++) s.tf[k] = (float)s.t[k];
}

// LDL^T solve of the 6x6 normal equations (upper triangle, row-major); false when a pivot is <= 1e-12 trace(A)
__device__ bool ldlt_solve(const double* up, const double* g, double* x)
{
    double A[6][6], L[6][6], d[6], y[6];
    int k = 0;
    for (int i = 0; i < 6; i++)
        for (int j = i; j < 6; j++) { A[i][j] = A[j][i] = up[k++]; }
    const double thr = 1e-12 * (A[0][0] + A[1][1] + A[2][2] + A[3][3] + A[4][4] + A[5][5]);
    for (int j = 0; j < 6; j++) {
        double dj = A[j][j];
        for (int m = 0; m < j; m++) dj -= L[j][m] * L[j][m] * d[m];
        if (!(dj > thr)) return false;
        d[j] = dj;
        L[j][j] = 1.0;
        for (int i = j + 1; i < 6; i++) {
            double a = A[i][j];
            for (int m = 0; m < j; m++) a -= L[i][m] * L[j][m] * d[m];
            L[i][j] = a / dj;
        }
    }
    for (int i = 0; i < 6; i++) {
        double a = g[i];
        for (int m = 0; m < i; m++) a -= L[i][m] * y[m];
        y[i] = a;
    }
    for (int i = 0; i < 6; i++) y[i] /= d[i];
    for (int i = 5; i >= 0; i--) {
        double a = y[i];
        for (int m = i + 1; m < 6; m++) a -= L[m][i] * x[m];
        x[i] = a;
    }
    return true;
}

// T <- exp(xi) T (Sophus SE3::exp, xi = (upsilon, omega)), quaternion renormalised
__device__ void apply_update(double* q, double* t, const double* xi)
{
    const double ux = xi[0], uy = xi[1], uz = xi[2], wx = xi[3], wy = xi[4], wz = xi[5];
    const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
    double k, B, Cc;
    if (th < 1e-4) { k = 0.5 - th2 / 48.0; B = 0.5 - th2 / 24.0; Cc = 1.0 / 6.0 - th2 / 120.0; }
    else { k = sin(0.5 * th) / th; B = (1.0 - cos(th)) / th2; Cc = (th - sin(th)) / (th2 * th); }
    const double dq[4] = {cos(0.5 * th), k * wx, k * wy, k * wz};
    const double cx = wy * uz - wz * uy, cy = wz * ux - wx * uz, cz = wx * uy - wy * ux;          // w x u
    const double ccx = wy * cz - wz * cy, ccy = wz * cx - wx * cz, ccz = wx * cy - wy * cx;       // w x (w x u)
    const double dt[3] = {ux + B * cx + Cc * ccx, uy + B * cy + Cc * ccy, uz + B * cz + Cc * ccz};
    double R[9], qn[4];
    quat_to_rot(dq, R);
    const double t0 = t[0], t1 = t[1], t2 = t[2];
    t[0] = R[0] * t0 + R[1] * t1 + R[2] * t2 + dt[0];
    t[1] = R[3] * t0 + R[4] * t1 + R[5] * t2 + dt[1];
    t[2] = R[6] * t0 + R[7] * t1 + R[8] * t2 + dt[2];
    quat_mul(dq, q, qn);
    quat_normalize(qn);
    for (int m = 0; m < 4; m++) q[m] = qn[m];
}

// the visibility grid of the points at the current pose: bounding box (order-independent min / max), then the nearest q_z per cell
__device__ void build_visibility(RefShared& s, const RefImage& im, const float* pts, int P, unsigned long long* zbuf)
{
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    double e[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
    for (int i = t; i < P; i += kRefThreads) {
        const double3 q = transform_d(s.Rd, s.t, make_float3(__ldg(pts + 3 * i), __ldg(pts + 3 * i + 1), __ldg(pts + 3 * i + 2)));
        if (!(q.z > im.znear && q.z < im.zfar)) continue;
        const double fu = im.fx * q.x / q.z + im.px, fv = im.fy * q.y / q.z + im.py;
        e[0] = fmin(e[0], fu); e[1] = fmax(e[1], fu); e[2] = fmin(e[2], fv); e[3] = fmax(e[3], fv);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        e[0] = fmin(e[0], __shfl_xor_sync(0xffffffffu, e[0], o)); e[1] = fmax(e[1], __shfl_xor_sync(0xffffffffu, e[1], o));
        e[2] = fmin(e[2], __shfl_xor_sync(0xffffffffu, e[2], o)); e[3] = fmax(e[3], __shfl_xor_sync(0xffffffffu, e[3], o));
    }
    if (lane == 0)
        for (int k = 0; k < 4; k++) s.ext[w][k] = e[k];
    __syncthreads();
    if (t == 0) {
        for (int k = 1; k < kRefWarps; k++) {
            e[0] = fmin(e[0], s.ext[k][0]); e[1] = fmax(e[1], s.ext[k][1]); e[2] = fmin(e[2], s.ext[k][2]); e[3] = fmax(e[3], s.ext[k][3]);
        }
        if (!(e[0] <= e[1])) {      // no point in the depth range: nothing is associated anyway
            s.grid = VisGrid{0.0, 0.0, 1.0, 1};
            s.ncells = 1;
        } else {
            const double bw = e[1] - e[0], bh = e[3] - e[2];
            const double side = fmax(fmax(sqrt(kVisPointsPerCell * bw * bh / P), fmax(bw, bh) / kVisMaxSide), 1.0);
            const int gw = (int)(bw / side) + 1, gh = (int)(bh / side) + 1;
            s.grid = VisGrid{e[0], e[2], side, gw};
            s.ncells = gw * gh;
        }
    }
    __syncthreads();
    for (int c = t; c < s.ncells; c += kRefThreads) zbuf[c] = 0x7FF0000000000000ull;     // +inf
    __syncthreads();
    const VisGrid g = s.grid;
    for (int i = t; i < P; i += kRefThreads) {
        const double3 q = transform_d(s.Rd, s.t, make_float3(__ldg(pts + 3 * i), __ldg(pts + 3 * i + 1), __ldg(pts + 3 * i + 2)));
        if (!(q.z > im.znear && q.z < im.zfar)) continue;
        atomicMin(zbuf + vis_cell(im, g, q), (unsigned long long)__double_as_longlong(q.z));      // q.z > 0: bit order = value order
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kHistThreads)
k_class_hist(const int32_t* __restrict__ label, int HW, int C, int* __restrict__ counts)
{
    extern __shared__ int hist[];
    for (int i = threadIdx.x; i < C; i += kHistThreads) hist[i] = 0;
    __syncthreads();
    const int32_t* L = label + (size_t)blockIdx.y * HW;
    const int lane = threadIdx.x & 31;
    for (int base = blockIdx.x * kHistThreads; base < HW; base += gridDim.x * kHistThreads) {
        const int p = base + threadIdx.x;
        const int l = p < HW ? __ldg(L + p) : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, l);
        if (l >= 0 && l < C && lane == __ffs(peers) - 1) atomicAdd(&hist[l], __popc(peers));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += kHistThreads)
        if (hist[i]) atomicAdd(&counts[(size_t)blockIdx.y * C + i], hist[i]);
}

struct RefineArgs {
    const int32_t* label;
    const float* depth;
    const float* meta;
    const float* rois;
    const float* poses;
    const int32_t* num_rows;
    const float* points;
    const int* counts;
    int num_meta, cap, C, P, B, H, W, batch_offset, min_pixels, iterations;
    float factor, znear, zfar, max_error;
    float* poses_refined;
    float* poses_icp;
    float* info;
    float* trace;
};

__global__ void __cluster_dims__(kRefHyp, 1, 1) __launch_bounds__(kRefThreads, 2)
k_pose_refine(const RefineArgs a)
{
    __shared__ RefShared s;
    __shared__ unsigned long long zbuf[kVisMaxCells];     // visibility grid; the score's pixel list reuses it
    int* sel = reinterpret_cast<int*>(zbuf);
    static_assert(kRefMaxPoints * sizeof(int) <= sizeof(zbuf), "pixel list must fit the grid's storage");
    cg::cluster_group cluster = cg::this_cluster();
    const int h = (int)cluster.block_rank();
    const int r = blockIdx.x / kRefHyp;
    const int t = threadIdx.x;
    const int nsteps = a.iterations + 1;
    float* trace = a.trace ? a.trace + ((size_t)r * kRefHyp + h) * nsteps * 8 : nullptr;

    const int nrows = a.num_rows ? min(max(__ldg(a.num_rows), 0), a.cap) : a.cap;
    const float* roi = a.rois + (size_t)r * 7;
    const int b = (int)roi[0] - a.batch_offset, c = (int)roi[1];
    const bool located = r < nrows && c > 0 && c < a.C && b >= 0 && b < a.B;
    const int n_mask = located ? a.counts[(size_t)b * a.C + c] : 0;
    if (!located || n_mask < a.min_pixels) {      // uniform over the cluster: no CTA waits at a cluster barrier
        if (h == 0 && t < 7) {
            a.poses_refined[(size_t)r * 7 + t] = 0.f;
            a.poses_icp[(size_t)r * 7 + t] = 0.f;
            if (t < 4) a.info[(size_t)r * 4 + t] = t == 0 ? (float)n_mask : 0.f;
        }
        if (trace)
            for (int i = t; i < nsteps * 8; i += kRefThreads) trace[i] = 0.f;
        return;
    }
    const float* m = a.meta + (size_t)b * a.num_meta;
    const RefImage im{a.label + (size_t)b * a.H * a.W, a.depth + (size_t)b * a.H * a.W, a.H, a.W, c, m[0], m[4], m[2], m[5],
                      a.factor, a.znear, a.zfar, a.max_error};
    const float* pts = a.points + (size_t)c * a.P * 3;
    auto point = [&](int i) { return make_float3(__ldg(pts + 3 * i), __ldg(pts + 3 * i + 1), __ldg(pts + 3 * i + 2)); };

    // ---- stage 1: mean depth offset of the inliers at the input pose, translation re-centred along its ray
    if (t == 0) {
        const float* p = a.poses + (size_t)r * 7;
        for (int k = 0; k < 4; k++) s.q[k] = p[k];
        quat_normalize(s.q);
        for (int k = 0; k < 3; k++) s.t[k] = p[4 + k];
        publish_pose(s);
    }
    __syncthreads();
    {
        build_visibility(s, im, pts, a.P, zbuf);
        double v[1] = {0.0};
        int cnt = 0;
        for (int i = t; i < a.P; i += kRefThreads) {
            const double3 q = transform_d(s.Rd, s.t, point(i));
            double3 X, n;
            double e;
            if (associate_d(im, s.grid, zbuf, q, X, n, e)) { v[0] += X.z - q.z; cnt++; }
        }
        block_sum<1>(s, v, cnt);
    }
    if (t == 0) {
        if (s.count > 0) {
            const double tz = s.t[2] + s.sum[0] / s.count;
            const double rx = s.t[2] == 0.0 ? 0.0 : s.t[0] / s.t[2], ry = s.t[2] == 0.0 ? 0.0 : s.t[1] / s.t[2];
            s.t[0] = rx * tz; s.t[1] = ry * tz; s.t[2] = tz;
        }
        for (int k = 0; k < 4; k++) s.q1[k] = s.q[k];
        for (int k = 0; k < 3; k++) s.t1[k] = s.t[k];
        s.t[2] += c_dz[h];
        s.stop = 0;
        publish_pose(s);
    }
    __syncthreads();

    // ---- stage 2: Gauss-Newton, re-associating all points at the current pose every step
    int done = 0;     // trace entries written
    for (int it = 0; it < a.iterations; it++) {
        build_visibility(s, im, pts, a.P, zbuf);
        double v[kRefSums];
#pragma unroll
        for (int k = 0; k < kRefSums; k++) v[k] = 0.0;
        int cnt = 0;
        for (int i = t; i < a.P; i += kRefThreads) {
            const double3 q = transform_d(s.Rd, s.t, point(i));
            double3 X, n;
            double e;
            if (!associate_d(im, s.grid, zbuf, q, X, n, e)) continue;
            const double w = 1.0 / X.z;
            const double J[6] = {w * n.x, w * n.y, w * n.z, w * (q.y * n.z - q.z * n.y), w * (q.z * n.x - q.x * n.z),
                                 w * (q.x * n.y - q.y * n.x)};
            const double ew = w * e;
            int k = 0;
#pragma unroll
            for (int i0 = 0; i0 < 6; i0++)
#pragma unroll
                for (int j0 = i0; j0 < 6; j0++) v[k++] += J[i0] * J[j0];
#pragma unroll
            for (int i0 = 0; i0 < 6; i0++) v[21 + i0] += J[i0] * ew;
            cnt++;
        }
        block_sum<kRefSums>(s, v, cnt);
        if (t == 0) {
            if (trace) {
                for (int k = 0; k < 4; k++) trace[it * 8 + k] = (float)s.q[k];
                for (int k = 0; k < 3; k++) trace[it * 8 + 4 + k] = (float)s.t[k];
                trace[it * 8 + 7] = (float)s.count;
            }
            double xi[6];
            if (s.count < kRefMinInliers || !ldlt_solve(s.sum, s.sum + 21, xi)) {
                s.stop = 1;
            } else {
                apply_update(s.q, s.t, xi);
                publish_pose(s);
            }
        }
        __syncthreads();
        if (s.stop) break;
        done = it + 1;
    }

    // ---- stage 3: distinct nearest live pixels within 1 cm (projective window), and the inliers at the final pose
    {
        build_visibility(s, im, pts, a.P, zbuf);
        int cnt = 0;
        for (int i = t; i < a.P; i += kRefThreads) {
            double3 X, n;
            double e;
            cnt += associate_d(im, s.grid, zbuf, transform_d(s.Rd, s.t, point(i)), X, n, e);
        }
        __syncthreads();      // the pixel list below overwrites the grid
        for (int i = t; i < a.P; i += kRefThreads) {
            const float3 q = transform(s.R, s.tf, point(i));
            int best = INT_MAX;
            if (q.z > im.znear && q.z < im.zfar) {
                const float fu = im.fx * q.x / q.z + im.px + 0.5f;
                const float fv = im.fy * q.y / q.z + im.py + 0.5f;
                if (fu >= 0.f && fu < (float)im.W && fv >= 0.f && fv < (float)im.H) {
                    const int u = (int)fu, v = (int)fv;
                    const int k = (int)ceilf(0.01f * im.fx / fmaxf(q.z - 0.01f, im.znear));
                    const int v0 = max(v - k, 0), v1 = min(v + k, im.H - 1), u0 = max(u - k, 0), u1 = min(u + k, im.W - 1);
                    float bd = 1e-4f;       // (1 cm)^2: strict
                    for (int y = v0; y <= v1; y++)
                        for (int x = u0; x <= u1; x++) {
                            float3 Xw;
                            if (!live_vertex(im, x, y, Xw)) continue;
                            const float dx = Xw.x - q.x, dy = Xw.y - q.y, dz = Xw.z - q.z;
                            const float d2 = dx * dx + dy * dy + dz * dz;
                            if (d2 < bd) { bd = d2; best = y * im.W + x; }
                        }
                }
            }
            sel[i] = best;
        }
        int np2 = 1;
        while (np2 < a.P) np2 <<= 1;
        for (int i = a.P + t; i < np2; i += kRefThreads) sel[i] = INT_MAX;
        __syncthreads();
        for (int k = 2; k <= np2; k <<= 1)          // bitonic sort, ascending
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = t; i < np2; i += kRefThreads) {
                    const int ixj = i ^ j;
                    if (ixj > i) {
                        const int x = sel[i], y = sel[ixj];
                        if ((x > y) == ((i & k) == 0)) { sel[i] = y; sel[ixj] = x; }
                    }
                }
                __syncthreads();
            }
        double v[1] = {0.0};
        int distinct = 0;
        for (int i = t; i < a.P; i += kRefThreads) distinct += sel[i] != INT_MAX && (i == 0 || sel[i] != sel[i - 1]);
        v[0] = cnt;
        block_sum<1>(s, v, distinct);
    }
    if (t == 0) {
        s.score = s.count;
        s.inliers = (int)s.sum[0];
        for (int k = 0; k < 4; k++) s.pose[k] = (float)s.q[k];
        for (int k = 0; k < 3; k++) s.pose[4 + k] = (float)s.t[k];
        if (trace)
            for (int it = done; it < nsteps; it++) {
                for (int k = 0; k < 7; k++) trace[it * 8 + k] = s.pose[k];
                trace[it * 8 + 7] = (float)s.inliers;
            }
    }
    cluster.sync();
    if (h == 0 && t == 0) {
        int best = 0, best_score = s.score;
        for (int k = 1; k < kRefHyp; k++) {
            const int sk = *cluster.map_shared_rank(&s.score, k);
            if (sk > best_score) { best = k; best_score = sk; }      // the first maximum
        }
        const RefShared* sb = cluster.map_shared_rank(&s, best);
        float* pr = a.poses_refined + (size_t)r * 7;
        float* pi = a.poses_icp + (size_t)r * 7;
        for (int k = 0; k < 4; k++) pr[k] = (float)s.q1[k];
        for (int k = 0; k < 3; k++) pr[4 + k] = (float)s.t1[k];
        for (int k = 0; k < 7; k++) pi[k] = sb->pose[k];
        float* inf = a.info + (size_t)r * 4;
        inf[0] = (float)n_mask;
        inf[1] = (float)best;
        inf[2] = (float)best_score / (float)a.P;
        inf[3] = (float)sb->inliers;
    }
    cluster.sync();      // rank 0 has read every CTA's shared memory
}

size_t refine_ws_bytes(int B, int C) { return align_up((size_t)B * C * sizeof(int), 256); }

}  // namespace pcnn

using namespace pcnn;

extern "C" int pcnn_pose_refine_workspace_bytes(int B, int C, size_t* bytes)
{
    PCNN_REQUIRE(bytes, "pose_refine: bytes is NULL");
    PCNN_REQUIRE(B >= 1 && C >= 2, "pose_refine: need B >= 1 and C >= 2 (got B = %d, C = %d)", B, C);
    *bytes = refine_ws_bytes(B, C);
    return PCNN_OK;
}

extern "C" int pcnn_pose_refine_fwd(const int32_t* label, const float* depth, const float* meta, int num_meta, const float* rois,
                                    const float* poses, const int32_t* num_rows, int cap, const float* points, int C, int P, int B,
                                    int H, int W, int batch_offset, float depth_factor, float znear, float zfar, float max_error,
                                    int min_pixels, int iterations, float* poses_refined, float* poses_icp, float* info,
                                    float* trace, void* workspace, size_t workspace_bytes, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    PCNN_REQUIRE(label && depth && meta && rois && poses && points && poses_refined && poses_icp && info && workspace,
                 "pose_refine: NULL required pointer");
    PCNN_REQUIRE(C >= 2 && C <= 4096, "pose_refine: C = %d outside [2, 4096]", C);
    PCNN_REQUIRE(P >= 1 && P <= kRefMaxPoints, "pose_refine: P = %d outside [1, %d]", P, kRefMaxPoints);
    PCNN_REQUIRE(iterations >= 0, "pose_refine: iterations = %d < 0", iterations);
    PCNN_REQUIRE(depth_factor > 0.f, "pose_refine: depth_factor must be > 0");
    PCNN_REQUIRE(znear < zfar, "pose_refine: need znear < zfar");
    PCNN_REQUIRE(B >= 1 && H >= 1 && W >= 1 && cap >= 0, "pose_refine: bad shape B = %d, H = %d, W = %d, cap = %d", B, H, W, cap);
    PCNN_REQUIRE(num_meta >= 6, "pose_refine: num_meta = %d < 6", num_meta);
    PCNN_REQUIRE((size_t)H * W <= (size_t)INT_MAX, "pose_refine: image too large");
    PCNN_REQUIRE(workspace_bytes >= refine_ws_bytes(B, C), "pose_refine: workspace %zu B < %zu B", workspace_bytes,
                 refine_ws_bytes(B, C));
    if (cap == 0) return PCNN_OK;
    int* counts = (int*)workspace;
    cudaError_t e = cudaMemsetAsync(counts, 0, (size_t)B * C * sizeof(int), stream);
    if (e != cudaSuccess) { set_error("pose_refine: memset: %s", cudaGetErrorString(e)); return PCNN_E_CUDA; }
    const int HW = H * W;
    const int per_image = max(1, min((HW + kHistThreads * 8 - 1) / (kHistThreads * 8), 64));
    k_class_hist<<<dim3(per_image, B), kHistThreads, C * sizeof(int), stream>>>(label, HW, C, counts);
    int rc = check_launch("pose_refine: class histogram");
    if (rc) return rc;
    RefineArgs args{label, depth, meta, rois, poses, num_rows, points, counts, num_meta, cap, C, P, B, H, W, batch_offset,
                    min_pixels, iterations, depth_factor, znear, zfar, max_error, poses_refined, poses_icp, info, trace};
    k_pose_refine<<<cap * kRefHyp, kRefThreads, 0, stream>>>(args);
    return check_launch("pose_refine");
}
