// evaluate.cu — scoring of the test-time records on the device (DESIGN.md §14): the segmentation confusion matrix of
// lib/datasets/imdb.py:123-125 (fast_hist) and the pose errors of lib/utils/pose_error.py (re, te, add, adi, reproj) over the
// (ground-truth object, detection of the same class) pairs of lib/datasets/lov.py:576-628 / linemod.py:700-760.
//
//   k_confusion     grid-stride over the pixels, four per lane (16-byte loads).  A warp whose 128 pixels all fall in one bin (the
//                   common case: label maps are spatially coherent) adds 128 once; otherwise __match_any_sync groups equal bins
//                   and the group's lowest lane adds its population.  Per-CTA uint32 bins in shared memory, flushed with one
//                   64-bit global atomic per non-empty bin.  Integer counts: the result does not depend on the order.
//   k_eval_pairs    one CTA: a warp per gt row counts the matching record rows with ballots, a block scan gives each gt its
//                   first pair slot, the warp then writes its pairs in ascending row order (gt-major: the reference's loop order).
//   k_eval_errors   persistent CTAs over the (pair, pose set) items: the estimate's rotation by quat2mat (fp64, rounded to fp32
//                   like the reference's float32 RT), re / te in fp64, then ADD or ADD-S and the reprojection error over the
//                   model points with fp64 per-thread sums and a fixed-order block reduction.  ADD-S stages the estimate's points
//                   in shared memory and searches the nearest one in fp32, then recomputes the winning distance in fp64.
// No host synchronisation and no allocation: the pair count stays on the device.
#include <limits.h>

#include "common.cuh"

namespace pcnn {

constexpr int kCmThreads = 512;
constexpr int kEvalMaxC = 128;
constexpr int kPairThreads = 1024;
constexpr int kPairItems = 4;
constexpr int kEvalMaxGt = kPairThreads * kPairItems;
constexpr int kErrThreads = 256;
constexpr int kEvalMaxPoints = 4096;
constexpr int kEvalRowFloats = 14;      // gt rows: batch, cls, [R | t] row-major
constexpr double kPixelThreshold = 5.0;  // linemod.py:732 `error_reprojection < 5`

// ------------------------------------------------------------------------------------------------------------------------------
// confusion matrix
__device__ __forceinline__ int cm_key(int g, int p, int C, unsigned& bad)
{
    if ((unsigned)p >= (unsigned)C) {       // a prediction outside [0, C) is an argument error, counted in status[0]
        bad++;
        return -1;
    }
    if ((unsigned)g >= (unsigned)C) return -1;   // imdb.py:124: k = (a >= 0) & (a < n)
    return g * C + p;
}

__global__ void __launch_bounds__(kCmThreads)
k_confusion(const int32_t* __restrict__ gt, const int32_t* __restrict__ pred, size_t n, int C, bool vec,
            unsigned long long* __restrict__ hist, unsigned long long* __restrict__ status)
{
    extern __shared__ unsigned s_bins[];   // [C*C]
    for (int i = threadIdx.x; i < C * C; i += kCmThreads) s_bins[i] = 0u;
    __syncthreads();
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    unsigned bad = 0;
    const size_t nv = vec ? n / 4 : 0;
    const size_t warp = ((size_t)blockIdx.x * kCmThreads + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * kCmThreads) >> 5;
    // warp-uniform trip count: every lane reaches the warp intrinsics with a full mask
    for (size_t base = warp * 32; base < nv; base += nwarps * 32) {
        const size_t i = base + lane;
        int k[4] = {-1, -1, -1, -1};
        if (i < nv) {
            const int4 a = __ldcs(reinterpret_cast<const int4*>(gt) + i);
            const int4 b = __ldcs(reinterpret_cast<const int4*>(pred) + i);
            k[0] = cm_key(a.x, b.x, C, bad); k[1] = cm_key(a.y, b.y, C, bad);
            k[2] = cm_key(a.z, b.z, C, bad); k[3] = cm_key(a.w, b.w, C, bad);
        }
        const bool same = k[0] == k[1] && k[0] == k[2] && k[0] == k[3];
        int uniform = 0;
        __match_all_sync(FULL, k[0], &uniform);
        if (__all_sync(FULL, same) && uniform) {
            if (lane == 0 && k[0] >= 0) atomicAdd(&s_bins[k[0]], 128u);
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const unsigned grp = __match_any_sync(FULL, k[j]);
                if (k[j] >= 0 && lane == __ffs(grp) - 1) atomicAdd(&s_bins[k[j]], (unsigned)__popc(grp));
            }
        }
    }
    for (size_t i = nv * 4 + (size_t)blockIdx.x * kCmThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kCmThreads) {
        const int k = cm_key(__ldg(gt + i), __ldg(pred + i), C, bad);
        if (k >= 0) atomicAdd(&s_bins[k], 1u);
    }
    for (int o = 16; o; o >>= 1) bad += __shfl_xor_sync(FULL, bad, o);
    if (lane == 0 && bad) atomicAdd(status, (unsigned long long)bad);
    __syncthreads();
    for (int i = threadIdx.x; i < C * C; i += kCmThreads)
        if (s_bins[i]) atomicAdd(hist + i, (unsigned long long)s_bins[i]);
}

// ------------------------------------------------------------------------------------------------------------------------------
// pose errors
struct EvalArgs {
    const float* gt;
    int num_gt;
    const float* rois;
    int roi_stride, cap;
    const int32_t* num_rows;
    const float* poses[4];
    int S;
    const float* meta;
    int num_meta, B, batch_offset;
    const float* points;
    int C, P;
    const float* symmetric;
    const float* threshold;
    const float* flip_z;
    int32_t* pairs;
    double* errors;
    int32_t* flags;
    int32_t* num_pairs;
    unsigned long long* counts;   // [S, 3, C]: count_all, count_correct, count_pixel
    unsigned long long* status;   // [2]: [1] += gt rows of a foreground class whose image is outside the batch, and num_rows outside [0, cap]
};

__device__ __forceinline__ bool gt_image(const EvalArgs& a, int j, int& b, int& cls)
{
    const float* g = a.gt + (size_t)j * kEvalRowFloats;
    b = (int)g[0];
    cls = (int)g[1];
    return cls > 0 && cls < a.C;   // lov.py:577 `cls_indexes[j] <= 0: continue`; classes past the table have no points
}

__global__ void __launch_bounds__(kPairThreads) k_eval_pairs(EvalArgs a)
{
    __shared__ int s_warp[kPairThreads / 32];
    __shared__ int s_cnt[kEvalMaxGt];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kPairThreads / 32;
    int nr = a.cap;
    if (a.num_rows) {
        const int v = *a.num_rows;
        nr = min(max(v, 0), a.cap);
        if (threadIdx.x == 0 && v != nr) atomicAdd(a.status + 1, 1ull);
    }
    for (int j = threadIdx.x; j < kEvalMaxGt; j += kPairThreads) s_cnt[j] = 0;
    __syncthreads();
    for (int j = warp; j < a.num_gt; j += nwarps) {
        int b, cls;
        if (!gt_image(a, j, b, cls)) continue;
        if (b - a.batch_offset < 0 || b - a.batch_offset >= a.B) {
            if (lane == 0) atomicAdd(a.status + 1, 1ull);
            continue;
        }
        if (lane < a.S) atomicAdd(a.counts + ((size_t)lane * 3 + 0) * a.C + cls, 1ull);   // lov.py:580
        int cnt = 0;
        for (int k0 = 0; k0 < nr; k0 += 32) {
            const int k = k0 + lane;
            const bool m = k < nr && (int)a.rois[(size_t)k * a.roi_stride] == b && (int)a.rois[(size_t)k * a.roi_stride + 1] == cls;
            cnt += __popc(__ballot_sync(FULL, m));
        }
        if (lane == 0) s_cnt[j] = cnt;
    }
    __syncthreads();
    // exclusive scan of s_cnt: serial over a thread's kPairItems entries, shuffles within the warp, then over the warp totals
    int run = 0;
#pragma unroll
    for (int i = 0; i < kPairItems; i++) run += s_cnt[threadIdx.x * kPairItems + i];
    int incl = run;
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += u;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = lane < nwarps ? s_warp[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(FULL, w, o);
            if (lane >= o) w += u;
        }
        if (lane < nwarps) s_warp[lane] = w;   // inclusive warp totals
    }
    __syncthreads();
    const int total = s_warp[nwarps - 1];
    int off = incl - run + (warp ? s_warp[warp - 1] : 0);
#pragma unroll
    for (int i = 0; i < kPairItems; i++) {
        const int c = s_cnt[threadIdx.x * kPairItems + i];
        s_cnt[threadIdx.x * kPairItems + i] = off;
        off += c;
    }
    if (threadIdx.x == 0) *a.num_pairs = total;
    __syncthreads();
    for (int j = warp; j < a.num_gt; j += nwarps) {
        int b, cls;
        if (!gt_image(a, j, b, cls) || b - a.batch_offset < 0 || b - a.batch_offset >= a.B) continue;
        int pos = s_cnt[j];
        for (int k0 = 0; k0 < nr; k0 += 32) {   // lov.py:582: rows in ascending order
            const int k = k0 + lane;
            const bool m = k < nr && (int)a.rois[(size_t)k * a.roi_stride] == b && (int)a.rois[(size_t)k * a.roi_stride + 1] == cls;
            const unsigned bal = __ballot_sync(FULL, m);
            if (m) {
                const int p = pos + __popc(bal & ((1u << lane) - 1u));
                a.pairs[2 * p] = j;
                a.pairs[2 * p + 1] = k;
            }
            pos += __popc(bal);
        }
    }
}

// transforms3d.quaternions.quat2mat (transforms3d 0.3.1, quaternions.py): normalise by |q|^2, identity below float64 eps
// (_FLOAT_EPS = np.finfo(np.float64).eps).  Evaluated in fp64 in the published operation order with the rounding intrinsics
// (never contracted into FMAs), then rounded to fp32 like the reference's float32 RT (lov.py:586-588).
__device__ __forceinline__ void quat2mat_f32(double w, double x, double y, double z, float* R)
{
    const double Nq = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(w, w), __dmul_rn(x, x)), __dmul_rn(y, y)), __dmul_rn(z, z));
    if (Nq < 2.220446049250313e-16) {   // `if Nq < _FLOAT_EPS: return np.eye(3)`
        for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.f : 0.f;
        return;
    }
    const double s = __ddiv_rn(2.0, Nq);
    const double X = __dmul_rn(x, s), Y = __dmul_rn(y, s), Z = __dmul_rn(z, s);
    const double wX = __dmul_rn(w, X), wY = __dmul_rn(w, Y), wZ = __dmul_rn(w, Z);
    const double xX = __dmul_rn(x, X), xY = __dmul_rn(x, Y), xZ = __dmul_rn(x, Z);
    const double yY = __dmul_rn(y, Y), yZ = __dmul_rn(y, Z), zZ = __dmul_rn(z, Z);
    R[0] = (float)__dsub_rn(1.0, __dadd_rn(yY, zZ)); R[1] = (float)__dsub_rn(xY, wZ); R[2] = (float)__dadd_rn(xZ, wY);
    R[3] = (float)__dadd_rn(xY, wZ); R[4] = (float)__dsub_rn(1.0, __dadd_rn(xX, zZ)); R[5] = (float)__dsub_rn(yZ, wX);
    R[6] = (float)__dsub_rn(xZ, wY); R[7] = (float)__dadd_rn(yZ, wX); R[8] = (float)__dsub_rn(1.0, __dadd_rn(xX, yY));
}

__global__ void k_gt_rows_from_blob(const float* __restrict__ blob, int n, float* __restrict__ rows)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* q = blob + (size_t)i * 13;
    float R[9];
    quat2mat_f32(q[6], q[7], q[8], q[9], R);
    float* o = rows + (size_t)i * kEvalRowFloats;
    o[0] = q[0];
    o[1] = q[1];
    for (int r = 0; r < 3; r++) {
        o[2 + 4 * r] = R[3 * r]; o[3 + 4 * r] = R[3 * r + 1]; o[4 + 4 * r] = R[3 * r + 2]; o[5 + 4 * r] = q[10 + r];
    }
}

// pose_error.re: angle of R_est inv(R_gt), clipped cosine; inv(R_gt) by the adjugate in fp64
__device__ __forceinline__ double rotation_error_deg(const float* Re, const double* Rg)
{
    const double c00 = Rg[4] * Rg[8] - Rg[5] * Rg[7], c01 = Rg[5] * Rg[6] - Rg[3] * Rg[8], c02 = Rg[3] * Rg[7] - Rg[4] * Rg[6];
    const double det = Rg[0] * c00 + Rg[1] * c01 + Rg[2] * c02;
    double inv[9];   // inv = adj / det, adj[i][j] = cofactor[j][i]
    inv[0] = c00; inv[3] = c01; inv[6] = c02;
    inv[1] = Rg[2] * Rg[7] - Rg[1] * Rg[8]; inv[4] = Rg[0] * Rg[8] - Rg[2] * Rg[6]; inv[7] = Rg[1] * Rg[6] - Rg[0] * Rg[7];
    inv[2] = Rg[1] * Rg[5] - Rg[2] * Rg[4]; inv[5] = Rg[2] * Rg[3] - Rg[0] * Rg[5]; inv[8] = Rg[0] * Rg[4] - Rg[1] * Rg[3];
    for (int i = 0; i < 9; i++) inv[i] /= det;
    double tr = 0.0;
    for (int i = 0; i < 3; i++)
        tr += (double)Re[3 * i] * inv[i] + (double)Re[3 * i + 1] * inv[3 + i] + (double)Re[3 * i + 2] * inv[6 + i];
    const double c = fmin(1.0, fmax(-1.0, 0.5 * (tr - 1.0)));
    return 180.0 * acos(c) / 3.141592653589793;
}

__device__ __forceinline__ float3 xform_f32(const float* R, const float* t, float x, float y, float z)
{
    return make_float3(__fadd_rn(fmaf(R[2], z, fmaf(R[1], y, R[0] * x)), t[0]),
                       __fadd_rn(fmaf(R[5], z, fmaf(R[4], y, R[3] * x)), t[1]),
                       __fadd_rn(fmaf(R[8], z, fmaf(R[7], y, R[6] * x)), t[2]));
}

__device__ __forceinline__ double3 xform_f64(const double* R, const double* t, float xf, float yf, float zf)
{
    const double x = xf, y = yf, z = zf;
    return make_double3(R[0] * x + R[1] * y + R[2] * z + t[0], R[3] * x + R[4] * y + R[5] * z + t[1],
                        R[6] * x + R[7] * y + R[8] * z + t[2]);
}

// pose_error.reproj's pixel of one point: K p in fp64, the quotient stored as float32 (`est = np.zeros((n, 2), np.float32)`)
__device__ __forceinline__ float2 project(const double* K, double x, double y, double z)
{
    const double u = K[0] * x + K[1] * y + K[2] * z, v = K[3] * x + K[4] * y + K[5] * z, w = K[6] * x + K[7] * y + K[8] * z;
    return make_float2((float)(u / w), (float)(v / w));
}

__global__ void __launch_bounds__(kErrThreads) k_eval_errors(EvalArgs a)
{
    extern __shared__ float4 s_est[];   // [P] the estimate's transformed points (ADD-S)
    __shared__ double s_red[2][kErrThreads];
    const int t = threadIdx.x;
    const int npairs = *a.num_pairs;
    const size_t maxp = (size_t)a.num_gt * a.cap;
    for (int it = blockIdx.x; it < npairs * a.S; it += gridDim.x) {
        const int p = it / a.S, s = it - p * a.S;
        const int j = a.pairs[2 * p], k = a.pairs[2 * p + 1];
        const float* g = a.gt + (size_t)j * kEvalRowFloats;
        const int cls = (int)g[1], b = (int)g[0] - a.batch_offset;
        double Rg[9], tg[3];
        for (int r = 0; r < 3; r++) {
            Rg[3 * r] = g[2 + 4 * r]; Rg[3 * r + 1] = g[3 + 4 * r]; Rg[3 * r + 2] = g[4 + 4 * r]; tg[r] = g[5 + 4 * r];
        }
        const float* q = a.poses[s] + (size_t)k * 7;
        float Re[9];
        quat2mat_f32(q[0], q[1], q[2], q[3], Re);
        const float te[3] = {q[4], q[5], q[6]};
        const double rerr = rotation_error_deg(Re, Rg);
        const double dx = tg[0] - te[0], dy = tg[1] - te[1], dz = tg[2] - te[2];
        const double terr = sqrt(dx * dx + dy * dy + dz * dz);
        // linemod.py:727-733: an eggbox estimate more than 90 degrees off is scored for reprojection as R diag(-1,-1,1)
        // (se3_mul(RT, RT_z): the first two columns negated, exact in float32), i.e. the model point (-x, -y, z)
        const float fs = (a.flip_z[cls] > 0.f && rerr > 90.0) ? -1.f : 1.f;
        const bool sym = a.symmetric[cls] > 0.f;
        double K[9];
        for (int i = 0; i < 9; i++) K[i] = a.meta[(size_t)b * a.num_meta + i];
        const float* pts = a.points + (size_t)cls * a.P * 3;
        double acc = 0.0, acc_px = 0.0;
        if (sym) {
            __syncthreads();   // the previous item's readers are done with s_est
            for (int i = t; i < a.P; i += kErrThreads) {
                const float3 e = xform_f32(Re, te, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
                s_est[i] = make_float4(e.x, e.y, e.z, 0.f);
            }
            __syncthreads();
        }
        for (int i = t; i < a.P; i += kErrThreads) {
            const float mx = pts[3 * i], my = pts[3 * i + 1], mz = pts[3 * i + 2];
            const double3 pg = xform_f64(Rg, tg, mx, my, mz);
            if (sym) {   // pose_error.adi: distance from each gt point to the nearest estimated point
                const float gx = (float)pg.x, gy = (float)pg.y, gz = (float)pg.z;
                float best = __int_as_float(0x7f800000);
                int bi = 0;
                for (int m = 0; m < a.P; m++) {
                    const float4 e = s_est[m];
                    const float ex = e.x - gx, ey = e.y - gy, ez = e.z - gz;
                    const float d2 = fmaf(ez, ez, fmaf(ey, ey, ex * ex));
                    if (d2 < best) { best = d2; bi = m; }
                }
                const float4 e = s_est[bi];
                const double ex = (double)e.x - pg.x, ey = (double)e.y - pg.y, ez = (double)e.z - pg.z;
                acc += sqrt(ex * ex + ey * ey + ez * ez);
            } else {     // pose_error.add
                const float3 e = xform_f32(Re, te, mx, my, mz);
                const double ex = (double)e.x - pg.x, ey = (double)e.y - pg.y, ez = (double)e.z - pg.z;
                acc += sqrt(ex * ex + ey * ey + ez * ez);
            }
            const float3 er = xform_f32(Re, te, fs * mx, fs * my, mz);
            const float2 pe = project(K, er.x, er.y, er.z), pq = project(K, pg.x, pg.y, pg.z);
            const double du = __fsub_rn(pe.x, pq.x), dv = __fsub_rn(pe.y, pq.y);
            acc_px += sqrt(du * du + dv * dv);
        }
        s_red[0][t] = acc;
        s_red[1][t] = acc_px;
        __syncthreads();
        for (int w = kErrThreads / 2; w > 0; w >>= 1) {
            if (t < w) {
                s_red[0][t] += s_red[0][t + w];
                s_red[1][t] += s_red[1][t + w];
            }
            __syncthreads();
        }
        if (t == 0) {
            const double add = s_red[0][0] / a.P, px = s_red[1][0] / a.P;
            double* e = a.errors + ((size_t)s * maxp + p) * 4;
            e[0] = rerr; e[1] = terr; e[2] = add; e[3] = px;
            const bool ok = add < (double)a.threshold[cls], ok_px = px < kPixelThreshold;   // lov.py:606, linemod.py:732
            a.flags[(size_t)s * maxp + p] = (ok ? 1 : 0) | (ok_px ? 2 : 0) | (fs < 0.f ? 4 : 0);
            if (ok) atomicAdd(a.counts + ((size_t)s * 3 + 1) * a.C + cls, 1ull);
            if (ok_px) atomicAdd(a.counts + ((size_t)s * 3 + 2) * a.C + cls, 1ull);
        }
        __syncthreads();   // s_red is reused by the next item
    }
}

}  // namespace pcnn

using namespace pcnn;

extern "C" int pcnn_eval_confusion(const int32_t* gt_label, const int32_t* label, size_t num_pixels, int C, int64_t* hist,
                                   int64_t* status, void* stream)
{
    PCNN_REQUIRE(gt_label && label && hist && status, "eval_confusion: null pointer");
    PCNN_REQUIRE(C >= 2 && C <= kEvalMaxC, "eval_confusion: C = %d (2 <= C <= %d)", C, kEvalMaxC);
    if (num_pixels == 0) return PCNN_OK;
    const bool vec = ((uintptr_t)gt_label % 16 == 0) && ((uintptr_t)label % 16 == 0);
    const int smem = C * C * (int)sizeof(unsigned);
    PCNN_SMEM_OPTIN(k_confusion, smem, "eval_confusion");
    // 8 four-pixel groups per thread at least; a CTA counts fewer than 2^31 pixels, so its uint32 bins cannot wrap
    size_t grid = (num_pixels + (size_t)kCmThreads * 32 - 1) / ((size_t)kCmThreads * 32);
    grid = grid < (size_t)kNumSMs * 4 ? grid : (size_t)kNumSMs * 4;
    const size_t min_grid = (num_pixels >> 31) + 1;
    grid = grid > min_grid ? grid : min_grid;
    PCNN_REQUIRE(grid <= INT_MAX, "eval_confusion: %zu pixels", num_pixels);
    k_confusion<<<(unsigned)grid, kCmThreads, smem, (cudaStream_t)stream>>>(gt_label, label, num_pixels, C, vec,
                                                                            (unsigned long long*)hist, (unsigned long long*)status);
    return check_launch("eval_confusion");
}

extern "C" int pcnn_eval_pose_errors(const float* gt_rows, int num_gt, const float* rois, int roi_stride, int cap,
                                     const int32_t* num_rows, const float* poses0, const float* poses1, const float* poses2,
                                     const float* poses3, int num_sets, const float* meta, int num_meta, int B, int batch_offset,
                                     const float* points, int C, int P, const float* symmetric, const float* threshold,
                                     const float* flip_z, int32_t* pairs, double* errors, int32_t* flags, int32_t* num_pairs,
                                     int64_t* counts, int64_t* status, void* stream)
{
    PCNN_REQUIRE(num_gt >= 0 && num_gt <= kEvalMaxGt, "eval_pose_errors: num_gt = %d (0 <= num_gt <= %d)", num_gt, kEvalMaxGt);
    PCNN_REQUIRE(cap >= 0 && roi_stride >= 2, "eval_pose_errors: cap = %d, roi_stride = %d (cap >= 0, roi_stride >= 2)", cap,
                 roi_stride);
    PCNN_REQUIRE((long long)num_gt * cap <= INT_MAX / 4, "eval_pose_errors: num_gt * cap = %lld pairs", (long long)num_gt * cap);
    PCNN_REQUIRE(num_sets >= 1 && num_sets <= 4, "eval_pose_errors: num_sets = %d (1 to 4 pose sets)", num_sets);
    const float* poses[4] = {poses0, poses1, poses2, poses3};
    for (int s = 0; s < num_sets; s++) PCNN_REQUIRE(poses[s] || cap == 0, "eval_pose_errors: pose set %d is null", s);
    PCNN_REQUIRE(C >= 2 && C <= kEvalMaxC, "eval_pose_errors: C = %d (2 <= C <= %d)", C, kEvalMaxC);
    PCNN_REQUIRE(P >= 1 && P <= kEvalMaxPoints, "eval_pose_errors: P = %d (1 <= P <= %d)", P, kEvalMaxPoints);
    PCNN_REQUIRE(B >= 1 && num_meta >= 9, "eval_pose_errors: B = %d, num_meta = %d (B >= 1, num_meta >= 9: K in meta[0:9])", B,
                 num_meta);
    PCNN_REQUIRE((gt_rows || num_gt == 0) && (rois || cap == 0) && meta && points && symmetric && threshold && flip_z,
                 "eval_pose_errors: null input");
    PCNN_REQUIRE(((pairs && errors && flags) || (long long)num_gt * cap == 0) && num_pairs && counts && status,
                 "eval_pose_errors: null output");
    EvalArgs a;
    a.gt = gt_rows; a.num_gt = num_gt; a.rois = rois; a.roi_stride = roi_stride; a.cap = cap; a.num_rows = num_rows;
    for (int s = 0; s < 4; s++) a.poses[s] = s < num_sets ? poses[s] : nullptr;
    a.S = num_sets; a.meta = meta; a.num_meta = num_meta; a.B = B; a.batch_offset = batch_offset; a.points = points;
    a.C = C; a.P = P; a.symmetric = symmetric; a.threshold = threshold; a.flip_z = flip_z; a.pairs = pairs; a.errors = errors;
    a.flags = flags; a.num_pairs = num_pairs; a.counts = (unsigned long long*)counts; a.status = (unsigned long long*)status;
    const int smem = P * (int)sizeof(float4);
    PCNN_SMEM_OPTIN(k_eval_errors, smem, "eval_pose_errors");
    cudaStream_t st = (cudaStream_t)stream;
    k_eval_pairs<<<1, kPairThreads, 0, st>>>(a);
    const long long items = (long long)num_gt * cap * num_sets;
    const int grid = (int)(items < kNumSMs * 4 ? (items > 0 ? items : 1) : kNumSMs * 4);
    k_eval_errors<<<grid, kErrThreads, smem, st>>>(a);
    return check_launch("eval_pose_errors");
}

extern "C" int pcnn_eval_gt_rows_from_blob(const float* pose_blob, int n, float* gt_rows, void* stream)
{
    PCNN_REQUIRE(n >= 0, "eval_gt_rows_from_blob: n = %d", n);
    PCNN_REQUIRE((pose_blob && gt_rows) || n == 0, "eval_gt_rows_from_blob: null pointer");
    if (n == 0) return PCNN_OK;
    k_gt_rows_from_blob<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(pose_blob, n, gt_rows);
    return check_launch("eval_gt_rows_from_blob");
}
