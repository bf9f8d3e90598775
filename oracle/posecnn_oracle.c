/*
 * posecnn_oracle.c — CPU restatement of the PoseCNN hot-path custom ops.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (posecnn_b200/) may
 * import, link or call this file; only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py use it, as the checker.
 *
 * The GPU kernels of the reference are the specification (the CPU kernels of the
 * same ops disagree with them, SURVEY.md finding 7).  Each function cites the
 * reference lines it restates (paths relative to /root/reference/lib).
 *
 * Arithmetic notes
 *  - nvcc (default -fmad=true) contracts `a*b + c*d` into fma(a, b, RN(c*d)) and
 *    `a*b + c` into fma(a, b, c); the restatement writes those fmaf() calls
 *    explicitly so that gcc reproduces the device rounding.  gcc is run with
 *    -ffp-contract=off so nothing else is fused.
 *  - float/double promotion follows the C++ source of the reference (e.g.
 *    `x - bb_width * (0.5 + scale)` is evaluated in double).
 *  - The reference Hough op is non-deterministic (atomicAdd compaction order,
 *    hough_voting_gpu_op.cu.cc:182-184); this oracle uses the canonical order of
 *    SURVEY.md §8(c): per-class pixel lists in ascending flat pixel index.
 *
 * Parity pinning: the reference ships no golden vectors (SURVEY.md §4).  This
 * oracle is pinned against the reference's own CUDA kernels, compiled unmodified
 * from a checkout of the reference behind a header shim (oracle/ref_shim,
 * oracle/ref_driver.cu -> oracle/_ref/libposecnn_ref.so) and run on the GPU;
 * tests/golden/ holds vectors produced that way (tests/golden/make_golden.py).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_ROI 128
#define VERTEX_CHANNELS 3

/* ------------------------------------------------------------------------- */
/* Hough voting — hough_voting_gpu_layer/hough_voting_gpu_op.cu.cc            */
/* ------------------------------------------------------------------------- */

/* angle_distance, .cu.cc:32-42 */
static inline float angle_distance_f(int cx, int cy, int x, int y, float u, float v, float n1)
{
    float dx = (float)(cx - x);
    float dy = (float)(cy - y);
    float n2 = sqrtf(fmaf(dx, dx, dy * dy));
    float dot = fmaf(u, dx, v * dy);
    return dot / (n1 * n2);
}

static inline double angle_distance_d(int cx, int cy, int x, int y, float u, float v)
{
    double dx = cx - x, dy = cy - y;
    double n1 = sqrt((double)u * u + (double)v * v);
    double n2 = sqrt(dx * dx + dy * dy);
    return ((double)u * dx + (double)v * dy) / (n1 * n2);
}

/* project_box, .cu.cc:84-120 */
static float project_box_f(int cls, const float* extents, const float* meta, float distance, float factor)
{
    float xHalf = (float)(extents[cls * 3 + 0] * 0.5);
    float yHalf = (float)(extents[cls * 3 + 1] * 0.5);
    float zHalf = (float)(extents[cls * 3 + 2] * 0.5);
    float bb[24];
    const float sx[8] = {1, -1, 1, -1, 1, -1, 1, -1};
    const float sy[8] = {1, 1, -1, -1, 1, 1, -1, -1};
    const float sz[8] = {1, 1, 1, 1, -1, -1, -1, -1};
    for (int i = 0; i < 8; i++) {
        bb[i * 3 + 0] = sx[i] * xHalf;
        bb[i * 3 + 1] = sy[i] * yHalf;
        bb[i * 3 + 2] = sz[i] * zHalf + distance;
    }
    float fx = meta[0], fy = meta[4], px = meta[2], py = meta[5];
    float minX = 1e8f, maxX = -1e8f, minY = 1e8f, maxY = -1e8f;
    for (int i = 0; i < 8; i++) {
        float x = fmaf(fx, bb[i * 3] / bb[i * 3 + 2], px);
        float y = fmaf(fy, bb[i * 3 + 1] / bb[i * 3 + 2], py);
        minX = fminf(minX, x);
        minY = fminf(minY, y);
        maxX = fmaxf(maxX, x);
        maxY = fmaxf(maxY, y);
    }
    float width = maxX - minX + 1;
    float height = maxY - minY + 1;
    return fmaxf(width, height) * factor;
}

float pcnn_oracle_project_box(int cls, const float* extents, const float* meta, float distance, float factor)
{
    return project_box_f(cls, extents, meta, distance, factor);
}

/* IoU, .cu.cc:73-82 */
static float iou_f(const float* a, const float* b)
{
    float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    float width = fmaxf(right - left + 1, 0.f), height = fmaxf(bottom - top + 1, 0.f);
    float interS = width * height;
    float Sa = (a[2] - a[0] + 1) * (a[3] - a[1] + 1);
    float Sb = (b[2] - b[0] + 1) * (b[3] - b[1] + 1);
    return interS / (Sa + Sb - interS);
}

/* compute_box_overlap, .cu.cc:123-172 (Eigen::Quaternionf::toRotationMatrix,
 * unit-quaternion form; 3x3 * 3x8 product evaluated coefficient-wise). */
static float box_overlap_f(int cls, const float* extents, const float* meta, const float* pose, const float* box)
{
    float xHalf = (float)(extents[cls * 3 + 0] * 0.5);
    float yHalf = (float)(extents[cls * 3 + 1] * 0.5);
    float zHalf = (float)(extents[cls * 3 + 2] * 0.5);
    const float sx[8] = {1, -1, 1, -1, 1, -1, 1, -1};
    const float sy[8] = {1, 1, -1, -1, 1, 1, -1, -1};
    const float sz[8] = {1, 1, 1, 1, -1, -1, -1, -1};
    float w = pose[6], x = pose[7], y = pose[8], z = pose[9];
    float tx = 2 * x, ty = 2 * y, tz = 2 * z;
    float twx = tx * w, twy = ty * w, twz = tz * w;
    float txx = tx * x, txy = ty * x, txz = tz * x;
    float tyy = ty * y, tyz = tz * y, tzz = tz * z;
    float R[9];
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
    float fx = meta[0], fy = meta[4], px = meta[2], py = meta[5];
    float x1 = 1e8f, x2 = -1e8f, y1 = 1e8f, y2 = -1e8f;
    for (int i = 0; i < 8; i++) {
        float bx = sx[i] * xHalf, by = sy[i] * yHalf, bz = sz[i] * zHalf;
        float X = fmaf(R[2], bz, fmaf(R[1], by, R[0] * bx)) + pose[10];
        float Y = fmaf(R[5], bz, fmaf(R[4], by, R[3] * bx)) + pose[11];
        float Z = fmaf(R[8], bz, fmaf(R[7], by, R[6] * bx)) + pose[12];
        float xx = fmaf(fx, X / Z, px);
        float yy = fmaf(fy, Y / Z, py);
        x1 = fminf(x1, xx); y1 = fminf(y1, yy);
        x2 = fmaxf(x2, xx); y2 = fmaxf(y2, yy);
    }
    float box_gt[4] = {x1, y1, x2, y2};
    return iou_f(box, box_gt);
}

typedef struct {
    int x, y;
    float u, v, n1, d, thr;
} sample_t;

/* votes for one class plane; returns nothing, fills votes[H*W] (float, integer valued)
 * and optionally ambig[H*W] (count of predicate evaluations within rounding distance
 * of a threshold, SURVEY.md §8(c) "predicate-boundary ambiguity"). .cu.cc:253-294 */
static void vote_plane(const sample_t* S, int ns, int H, int W, float inlier, float* votes, int* ambig)
{
#pragma omp parallel for schedule(dynamic, 4)
    for (int cy = 0; cy < H; cy++) {
        for (int cx = 0; cx < W; cx++) {
            int cnt = 0, amb = 0;
            for (int i = 0; i < ns; i++) {
                const sample_t* s = &S[i];
                float dxa = fabsf((float)(s->x - cx));
                float dya = fabsf((float)(s->y - cy));
                int in_win = (dxa < s->thr) && (dya < s->thr);
                int near_win = 0;
                if (ambig) {
                    float tol = 1e-4f * s->thr;
                    near_win = (fabsf(dxa - s->thr) < tol && dya < s->thr + tol) ||
                               (fabsf(dya - s->thr) < tol && dxa < s->thr + tol);
                }
                if (!in_win && !near_win) continue;
                float c = angle_distance_f(cx, cy, s->x, s->y, s->u, s->v, s->n1);
                if (ambig) {
                    double cd = angle_distance_d(cx, cy, s->x, s->y, s->u, s->v);
                    if (fabs(cd - (double)inlier) < 1e-6) amb++;
                    else if (near_win && cd > inlier) amb++;
                }
                if (in_win && c > inlier) cnt++;
            }
            votes[cy * W + cx] = (float)cnt;
            if (ambig) ambig[cy * W + cx] = amb;
        }
    }
}

/* Exactness criterion of the interval scan (DESIGN.md §3.3).  The device op represents the vote set of one (sample,
 * row) pair as one interval of cells, the pixel's own row as one whole side of its window.  `pass[i]` is the
 * reference predicate at cell wmin + i of the window row; the pair is exact when its set has that form (or is empty),
 * irregular otherwise (the fp32 predicate is not monotone along the row there). */
int pcnn_oracle_hough_row_exact(const unsigned char* pass, int wmin, int wmax, int x, int own_row)
{
    int n = wmax - wmin + 1, first = -1, last = -1, count = 0;
    for (int i = 0; i < n; i++)
        if (pass[i]) {
            if (first < 0) first = i;
            last = i;
            count++;
        }
    if (count == 0) return 1;
    if (count != last - first + 1) return 0;
    if (!own_row) return 1;
    /* own row: exactly the cells x+1 .. wmax or wmin .. x-1 */
    return (wmin + first == x + 1 && wmin + last == wmax) || (wmin + first == wmin && wmin + last == x - 1);
}

/* slack[H*W]: for each cell, the number of irregular (sample, row) pairs whose window row contains it; pairs[0] =
 * (sample, row) pairs inside a window, pairs[1] = irregular ones.  Same predicate and window test as vote_plane. */
static void slack_plane(const sample_t* S, int ns, int H, int W, float inlier, int* slack, long long* pairs)
{
    long long np = 0, nirr = 0;
#pragma omp parallel reduction(+ : np, nirr)
    {
        unsigned char* pass = (unsigned char*)malloc((size_t)W);
#pragma omp for schedule(dynamic, 4)
        for (int cy = 0; cy < H; cy++) {
            int* srow = slack + (size_t)cy * W;
            memset(srow, 0, sizeof(int) * (size_t)W);
            for (int i = 0; i < ns; i++) {
                const sample_t* s = &S[i];
                if (!(fabsf((float)(s->y - cy)) < s->thr)) continue;
                int wmin = s->x, wmax = s->x;
                if (!(0.f < s->thr)) continue;
                while (wmin > 0 && fabsf((float)(s->x - (wmin - 1))) < s->thr) wmin--;
                while (wmax < W - 1 && fabsf((float)(s->x - (wmax + 1))) < s->thr) wmax++;
                for (int cx = wmin; cx <= wmax; cx++)
                    pass[cx - wmin] = angle_distance_f(cx, cy, s->x, s->y, s->u, s->v, s->n1) > inlier;
                np++;
                if (!pcnn_oracle_hough_row_exact(pass, wmin, wmax, s->x, cy == s->y)) {
                    nirr++;
                    for (int cx = wmin; cx <= wmax; cx++) srow[cx]++;
                }
            }
        }
        free(pass);
    }
    pairs[0] = np;
    pairs[1] = nirr;
}

/* hough_data for one cell, .cu.cc:296-331.  dist accumulated sequentially in the
 * canonical sample order. */
static void cell_data(const sample_t* S, int ns, int cls, const float* extents, const float* meta, int cx, int cy,
                      float inlier, float* out_dist, float* out_h2, float* out_w2, float* out_votes)
{
    float distance = 0, votes = 0;
    for (int i = 0; i < ns; i++) {
        const sample_t* s = &S[i];
        if (angle_distance_f(cx, cy, s->x, s->y, s->u, s->v, s->n1) > inlier) {
            float dx = fabsf((float)(s->x - cx)), dy = fabsf((float)(s->y - cy));
            if (dx < s->thr && dy < s->thr) { votes += 1; distance += s->d; }
        }
    }
    *out_votes = votes;
    if (!(votes > 0)) { *out_dist = 0; *out_h2 = 0; *out_w2 = 0; return; }
    distance /= votes;
    float bbw = -1, bbh = -1;
    float thr2 = project_box_f(cls, extents, meta, distance, 0.6f);
    for (int i = 0; i < ns; i++) {
        const sample_t* s = &S[i];
        if (angle_distance_f(cx, cy, s->x, s->y, s->u, s->v, s->n1) > inlier) {
            float dx = fabsf((float)(s->x - cx)), dy = fabsf((float)(s->y - cy));
            if (dx > bbw && dx < thr2 && dy < thr2) bbw = dx;
            if (dy > bbh && dx < thr2 && dy < thr2) bbh = dy;
        }
    }
    *out_dist = distance; *out_h2 = 2 * bbh; *out_w2 = 2 * bbw;
}

/* compute_rois_kernel, .cu.cc:386-576: one maximum -> 1 (test) or 9 (train) rows. */
static void emit_rows(int roi_index, int is_train, int batch_index, int cls, int x, int y, float votes, float bb_distance,
                      float bb_height, float bb_width, const float* extents, const float* meta, const float* gt,
                      int num_gt, int C, float* top_box, float* top_pose, float* top_target, float* top_weight,
                      int* top_domain)
{
    float scale = 0.05f;
    float fx = meta[0], fy = meta[4], px = meta[2], py = meta[5];
    float rx = (x - px) / fx;
    float ry = (y - py) / fy;
    float* b0 = top_box + (size_t)roi_index * 7;
    b0[0] = (float)batch_index;
    b0[1] = (float)cls;
    b0[2] = (float)(x - bb_width * (0.5 + scale));
    b0[3] = (float)(y - bb_height * (0.5 + scale));
    b0[4] = (float)(x + bb_width * (0.5 + scale));
    b0[5] = (float)(y + bb_height * (0.5 + scale));
    b0[6] = votes;
    int nrow = is_train ? 9 : 1;
    for (int i = 0; i < nrow; i++) {
        float* p = top_pose + (size_t)(roi_index + i) * 7;
        p[0] = 1; p[1] = 0; p[2] = 0; p[3] = 0;
        p[4] = rx * bb_distance; p[5] = ry * bb_distance; p[6] = bb_distance;
        if (is_train) top_domain[roi_index + i] = (num_gt == 0) ? 1 : 0;
    }
    if (!is_train) return;
    for (int i = 0; i < num_gt; i++) {
        int gt_batch = (int)gt[i * 13 + 0];
        int gt_id = (int)gt[i * 13 + 1];
        if (cls == gt_id && batch_index == gt_batch) {
            float overlap = box_overlap_f(cls, extents, meta, gt + i * 13, b0 + 2);
            if (overlap > 0.2f) {
                for (int j = 0; j < 9; j++)
                    for (int k = 0; k < 4; k++) {
                        top_target[(size_t)(roi_index + j) * 4 * C + 4 * cls + k] = gt[i * 13 + 6 + k];
                        top_weight[(size_t)(roi_index + j) * 4 * C + 4 * cls + k] = 1;
                    }
                break;
            }
        }
    }
    float x1 = b0[2], y1 = b0[3], x2 = b0[4], y2 = b0[5];
    float ww = x2 - x1, hh = y2 - y1;
    /* jitter order .cu.cc:476-554 */
    const int jx[8] = {-1, 1, -1, 1, 0, -1, 0, 1};
    const int jy[8] = {-1, -1, 1, 1, -1, 0, 1, 0};
    for (int j = 0; j < 8; j++) {
        float* b = top_box + (size_t)(roi_index + 1 + j) * 7;
        b[0] = (float)batch_index;
        b[1] = (float)cls;
        b[2] = jx[j] == 0 ? x1 : (float)(x1 + jx[j] * (0.05 * ww));
        b[3] = jy[j] == 0 ? y1 : (float)(y1 + jy[j] * (0.05 * hh));
        b[4] = b[2] + ww;
        b[5] = b[3] + hh;
        b[6] = votes;
    }
}

/*
 * Whole op: HoughvotinggpuOp<GpuDevice>::Compute, hough_voting_gpu_op.cc:321-428 and
 * HoughVotingLaucher, .cu.cc:615-797.  Output buffers must hold MAX_ROI*9 = 1152 rows
 * and are zero-filled here (reset_outputs, .cu.cc:579-588).  *num_rois receives the
 * emitted row count (the op then reports max(1, num_rois) rows, .cc:379-383).
 * votes_dbg / ambig_dbg: optional [B][C][H][W] planes (zero for classes not voted).
 * slack_dbg / pairs_dbg: optional [B][C][H][W] slack planes and [B][C][2] pair counts of slack_plane (both or neither).
 */
int pcnn_oracle_hough(const int* label, const float* vertex, const float* extents, const float* meta_all,
                      const float* gt, int B, int H, int W, int C, int num_gt, int num_meta, int is_train,
                      float inlier, int label_thr, float vote_thr, float per_thr, int skip, float* top_box,
                      float* top_pose, float* top_target, float* top_weight, int* top_domain, int* num_rois,
                      float* votes_dbg, int* ambig_dbg, int* slack_dbg, long long* pairs_dbg)
{
    const int cap_rows = MAX_ROI * 9;
    memset(top_box, 0, sizeof(float) * cap_rows * 7);
    memset(top_pose, 0, sizeof(float) * cap_rows * 7);
    memset(top_target, 0, sizeof(float) * cap_rows * 4 * C);
    memset(top_weight, 0, sizeof(float) * cap_rows * 4 * C);
    memset(top_domain, 0, sizeof(int) * cap_rows);
    if (votes_dbg) memset(votes_dbg, 0, sizeof(float) * (size_t)B * C * H * W);
    if (ambig_dbg) memset(ambig_dbg, 0, sizeof(int) * (size_t)B * C * H * W);
    if (slack_dbg) memset(slack_dbg, 0, sizeof(int) * (size_t)B * C * H * W);
    if (pairs_dbg) memset(pairs_dbg, 0, sizeof(long long) * (size_t)B * C * 2);
    int nrois = 0;
    int index_size = B > 0 ? MAX_ROI / B : 0; /* .cu.cc:733 */
    int HW = H * W;
    int* sizes = (int*)malloc(sizeof(int) * C);
    sample_t* S = (sample_t*)malloc(sizeof(sample_t) * (size_t)HW);
    float* votes = (float*)malloc(sizeof(float) * (size_t)HW);
    int* amb = ambig_dbg ? (int*)malloc(sizeof(int) * (size_t)HW) : NULL;

    for (int n = 0; n < B; n++) {
        const int* lab = label + (size_t)n * HW;
        const float* vert = vertex + (size_t)n * HW * VERTEX_CHANNELS * C;
        const float* meta = meta_all + (size_t)n * num_meta;
        memset(sizes, 0, sizeof(int) * C);
        for (int p = 0; p < HW; p++) {
            int c = lab[p];
            if (c > 0 && c < C) sizes[c]++;
        }
        /* candidate maxima of this image in canonical (class slot, flat cell) order */
        int nmax = 0;
        int max_cls[MAX_ROI], max_x[MAX_ROI], max_y[MAX_ROI];
        float max_votes[MAX_ROI], max_dist[MAX_ROI], max_h2[MAX_ROI], max_w2[MAX_ROI];
        for (int c = 1; c < C && nmax < index_size; c++) {
            if (sizes[c] <= label_thr) continue; /* .cu.cc:656 */
            /* canonical pixel list, sampled every `skip` (.cu.cc:269) */
            int rank = 0, ns = 0;
            for (int p = 0; p < HW; p++) {
                if (lab[p] != c) continue;
                if (rank % skip == 0) {
                    sample_t* s = &S[ns++];
                    s->x = p % W;
                    s->y = p / W;
                    size_t off = (size_t)VERTEX_CHANNELS * c + (size_t)VERTEX_CHANNELS * C * p;
                    s->u = vert[off];
                    s->v = vert[off + 1];
                    s->d = expf(vert[off + 2]);
                    s->n1 = sqrtf(fmaf(s->u, s->u, s->v * s->v));
                    s->thr = project_box_f(c, extents, meta, s->d, 0.6f);
                }
                rank++;
            }
            vote_plane(S, ns, H, W, inlier, votes, amb);
            if (votes_dbg) memcpy(votes_dbg + ((size_t)n * C + c) * HW, votes, sizeof(float) * HW);
            if (ambig_dbg) memcpy(ambig_dbg + ((size_t)n * C + c) * HW, amb, sizeof(int) * HW);
            if (slack_dbg)
                slack_plane(S, ns, H, W, inlier, slack_dbg + ((size_t)n * C + c) * HW, pairs_dbg + ((size_t)n * C + c) * 2);
            if (vote_thr > 0) {
                /* compute_max_indexes_kernel, .cu.cc:335-383 (canonical: ascending flat index) */
                for (int p = 0; p < HW && nmax < index_size; p++) {
                    if (!(votes[p] > vote_thr)) continue;
                    int cx = p % W, cy = p / W, flag = 0;
                    for (int x = cx - 3; x <= cx + 3 && !flag; x++)
                        for (int y = cy - 3; y <= cy + 3; y++)
                            if (x >= 0 && x < W && y >= 0 && y < H && votes[y * W + x] > votes[p]) { flag = 1; break; }
                    if (flag) continue;
                    float dist, h2, w2, vv;
                    cell_data(S, ns, c, extents, meta, cx, cy, inlier, &dist, &h2, &w2, &vv);
                    if (!(h2 > 0 && w2 > 0)) continue;
                    if (votes[p] / (h2 * w2) < per_thr) continue;
                    max_cls[nmax] = c; max_x[nmax] = cx; max_y[nmax] = cy;
                    max_votes[nmax] = votes[p]; max_dist[nmax] = dist; max_h2[nmax] = h2; max_w2[nmax] = w2;
                    nmax++;
                }
            } else {
                /* thrust::max_element: first maximal element, .cu.cc:756 */
                int best = 0;
                for (int p = 1; p < HW; p++)
                    if (votes[p] > votes[best]) best = p;
                float dist, h2, w2, vv;
                cell_data(S, ns, c, extents, meta, best % W, best / W, inlier, &dist, &h2, &w2, &vv);
                max_cls[nmax] = c; max_x[nmax] = best % W; max_y[nmax] = best / W;
                max_votes[nmax] = votes[best]; max_dist[nmax] = dist; max_h2[nmax] = h2; max_w2[nmax] = w2;
                nmax++;
            }
        }
        for (int i = 0; i < nmax; i++) {
            emit_rows(nrois, is_train, n, max_cls[i], max_x[i], max_y[i], max_votes[i], max_dist[i], max_h2[i],
                      max_w2[i], extents, meta, gt, num_gt, C, top_box, top_pose, top_target, top_weight, top_domain);
            nrois += is_train ? 9 : 1;
        }
    }
    *num_rois = nrois;
    free(sizes); free(S); free(votes); free(amb);
    return 0;
}

/* ------------------------------------------------------------------------- */
/* RoiPool — roi_pooling_layer/roi_pooling_op_gpu.cu.cc:19-101, 134-229       */
/* ------------------------------------------------------------------------- */
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

int pcnn_oracle_roi_pool_fwd(const float* bottom, const float* rois, int num_rois, int channel_rois, int height,
                             int width, int channels, int ph_n, int pw_n, float spatial_scale, int pool_channel,
                             float* top, int* argmax)
{
    int cout = pool_channel ? 1 : channels;
    for (int n = 0; n < num_rois; n++) {
        const float* r = rois + (size_t)n * channel_rois;
        int b = (int)r[0], roi_cls = (int)r[1];
        int rsw = (int)roundf(r[2] * spatial_scale), rsh = (int)roundf(r[3] * spatial_scale);
        int rew = (int)roundf(r[4] * spatial_scale), reh = (int)roundf(r[5] * spatial_scale);
        int rw = imax(rew - rsw + 1, 1), rh = imax(reh - rsh + 1, 1);
        float bh = (float)rh / (float)ph_n, bw = (float)rw / (float)pw_n;
        const float* img = bottom + (size_t)b * channels * height * width;
        for (int ph = 0; ph < ph_n; ph++)
            for (int pw = 0; pw < pw_n; pw++) {
                int hs = (int)floorf((float)ph * bh), ws = (int)floorf((float)pw * bw);
                int he = (int)ceilf((float)(ph + 1) * bh), we = (int)ceilf((float)(pw + 1) * bw);
                hs = imin(imax(hs + rsh, 0), height); he = imin(imax(he + rsh, 0), height);
                ws = imin(imax(ws + rsw, 0), width);  we = imin(imax(we + rsw, 0), width);
                int empty = (he <= hs) || (we <= ws);
                for (int c = 0; c < cout; c++) {
                    int cc = pool_channel ? roi_cls : c;
                    float maxval = empty ? 0 : -FLT_MAX;
                    int maxidx = -1;
                    for (int h = hs; h < he; h++)
                        for (int w = ws; w < we; w++) {
                            int bi = (h * width + w) * channels + cc;
                            if (img[bi] > maxval) { maxval = img[bi]; maxidx = bi; }
                        }
                    size_t o = (((size_t)n * ph_n + ph) * pw_n + pw) * cout + c;
                    top[o] = maxval;
                    argmax[o] = maxidx;
                }
            }
    }
    return 0;
}

int pcnn_oracle_roi_pool_bwd(const float* top_diff, const int* argmax, const float* rois, int batch, int num_rois,
                             int channel_rois, int height, int width, int channels, int ph_n, int pw_n,
                             float spatial_scale, int pool_channel, float* bottom_diff)
{
#pragma omp parallel for
    for (int n = 0; n < batch; n++)
        for (int h = 0; h < height; h++)
            for (int w = 0; w < width; w++)
                for (int c = 0; c < channels; c++) {
                    float g = 0;
                    for (int rn = 0; rn < num_rois; rn++) {
                        const float* r = rois + (size_t)rn * channel_rois;
                        if (n != (int)r[0]) continue;
                        if (pool_channel && c != (int)r[1]) continue;
                        int rsw = (int)roundf(r[2] * spatial_scale), rsh = (int)roundf(r[3] * spatial_scale);
                        int rew = (int)roundf(r[4] * spatial_scale), reh = (int)roundf(r[5] * spatial_scale);
                        if (!(w >= rsw && w <= rew && h >= rsh && h <= reh)) continue;
                        size_t off = (size_t)rn * ph_n * pw_n * (pool_channel ? 1 : channels);
                        int rw = imax(rew - rsw + 1, 1), rh = imax(reh - rsh + 1, 1);
                        float bh = (float)rh / (float)ph_n, bw = (float)rw / (float)pw_n;
                        int phs = (int)floorf((float)(h - rsh) / bh), phe = (int)ceilf((float)(h - rsh + 1) / bh);
                        int pws = (int)floorf((float)(w - rsw) / bw), pwe = (int)ceilf((float)(w - rsw + 1) / bw);
                        phs = imin(imax(phs, 0), ph_n); phe = imin(imax(phe, 0), ph_n);
                        pws = imin(imax(pws, 0), pw_n); pwe = imin(imax(pwe, 0), pw_n);
                        for (int ph = phs; ph < phe; ph++)
                            for (int pw = pws; pw < pwe; pw++) {
                                size_t o = pool_channel ? off + (size_t)ph * pw_n + pw
                                                        : off + ((size_t)ph * pw_n + pw) * channels + c;
                                if (argmax[o] == (h * width + w) * channels + c) g += top_diff[o];
                            }
                    }
                    bottom_diff[(((size_t)n * height + h) * width + w) * channels + c] = g;
                }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* Hardlabel — hard_label_layer/hard_label_op_gpu.cu.cc:16-29                 */
/* ------------------------------------------------------------------------- */
int pcnn_oracle_hard_label(const float* prob, const int* gt, long npix, int C, float threshold, float* top)
{
    for (long p = 0; p < npix; p++) {
        for (int c = 0; c < C; c++) top[p * C + c] = 0.f;
        int g = gt[p];
        if (g != -1 && (g > 0 || prob[p * C + g] < threshold)) top[p * C + g] = 1.f;
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* Project — projecting_layer/projecting_op_gpu.cu.cc:16-73 (fwd), 101-169    */
/* Backproject — backprojecting_layer/backprojecting_op_gpu.cu.cc:16-126,158-217 */
/* ------------------------------------------------------------------------- */

/* pixel -> voxel (shared by ProjectForward and BackprojectBackward).  near_half is
 * set when a pre-round coordinate is within 1e-3 of a half integer (round() tie zone). */
static inline int pixel_to_voxel(const float* m, int w, int h, float depth, int G, int* vd, int* vh, int* vw,
                                 int* near_half)
{
    float RX = fmaf(m[9], (float)w, m[10] * (float)h) + m[11];
    float RY = fmaf(m[12], (float)w, m[13] * (float)h) + m[14];
    float RZ = fmaf(m[15], (float)w, m[16] * (float)h) + m[17];
    float X = depth * RX, Y = depth * RY, Z = depth * RZ;
    float X1 = fmaf(m[32], Z, fmaf(m[30], X, m[31] * Y)) + m[33];
    float Y1 = fmaf(m[36], Z, fmaf(m[34], X, m[35] * Y)) + m[37];
    float Z1 = fmaf(m[40], Z, fmaf(m[38], X, m[39] * Y)) + m[41];
    float a = (X1 - m[45]) / m[42], b = (Y1 - m[46]) / m[43], c = (Z1 - m[47]) / m[44];
    *vd = (int)roundf(a); *vh = (int)roundf(b); *vw = (int)roundf(c);
    if (near_half) {
        float fa = fabsf(a - floorf(a) - 0.5f), fb = fabsf(b - floorf(b) - 0.5f), fc = fabsf(c - floorf(c) - 0.5f);
        *near_half = (fa < 1e-3f) || (fb < 1e-3f) || (fc < 1e-3f);
    }
    return *vd >= 0 && *vd < G && *vh >= 0 && *vh < G && *vw >= 0 && *vw < G;
}

/* voxel -> pixel (shared by BackprojectForward and ProjectBackward) */
static inline void voxel_to_pixel(const float* m, int d, int h, int w, int* px, int* py, float* Z1out, int* near_half)
{
    float X = fmaf((float)d, m[42], m[45]);
    float Y = fmaf((float)h, m[43], m[46]);
    float Z = fmaf((float)w, m[44], m[47]);
    float X1 = fmaf(m[20], Z, fmaf(m[18], X, m[19] * Y)) + m[21];
    float Y1 = fmaf(m[24], Z, fmaf(m[22], X, m[23] * Y)) + m[25];
    float Z1 = fmaf(m[28], Z, fmaf(m[26], X, m[27] * Y)) + m[29];
    float x1 = fmaf(m[2], Z1, fmaf(m[0], X1, m[1] * Y1));
    float x2 = fmaf(m[5], Z1, fmaf(m[3], X1, m[4] * Y1));
    float x3 = fmaf(m[8], Z1, fmaf(m[6], X1, m[7] * Y1));
    float a = x1 / x3, b = x2 / x3;
    *px = (int)roundf(a); *py = (int)roundf(b);
    *Z1out = Z1;
    if (near_half) {
        float fa = fabsf(a - floorf(a) - 0.5f), fb = fabsf(b - floorf(b) - 0.5f);
        *near_half = (fa < 1e-3f) || (fb < 1e-3f) || !(fabsf(a) < 1e7f) || !(fabsf(b) < 1e7f);
    }
}

/* gather: out[B,H,W,Cf] = vox[B,G,G,G,Cf] at the voxel hit by the pixel, else 0.
 * ProjectForward (data=bottom_data) and BackprojectBackward (data=top_diff). */
int pcnn_oracle_pixel_gather(const float* vox, const float* depth, const float* meta, int B, int H, int W, int Cf,
                             int num_meta, int G, float* out, unsigned char* ambig)
{
#pragma omp parallel for
    for (int n = 0; n < B; n++)
        for (int h = 0; h < H; h++)
            for (int w = 0; w < W; w++) {
                size_t pix = ((size_t)n * H + h) * W + w;
                int vd, vh, vw, nh;
                int inside = pixel_to_voxel(meta + (size_t)n * num_meta, w, h, depth[pix], G, &vd, &vh, &vw, &nh);
                if (ambig) ambig[pix] = (unsigned char)nh;
                for (int c = 0; c < Cf; c++)
                    out[pix * Cf + c] =
                        inside ? vox[((((size_t)n * G + vd) * G + vh) * G + vw) * Cf + c] : 0.f;
            }
    return 0;
}

/* window average around the projected voxel.  BackprojectForward (with labels/flag) and
 * ProjectBackward (data only; no division when count==0 is the same as dividing 0). */
int pcnn_oracle_voxel_average(const float* data, const float* label, const float* depth, const float* meta,
                              const float* label_3d, int B, int H, int W, int Cf, int C, int num_meta, int G, int ks,
                              float threshold, float* top_data, float* top_label, float* top_flag,
                              unsigned char* ambig)
{
#pragma omp parallel for collapse(2)
    for (int n = 0; n < B; n++)
        for (int d = 0; d < G; d++)
            for (int h = 0; h < G; h++)
                for (int w = 0; w < G; w++) {
                    size_t v = (((size_t)n * G + d) * G + h) * G + w;
                    int px, py, nh;
                    float Z1;
                    voxel_to_pixel(meta + (size_t)n * num_meta, d, h, w, &px, &py, &Z1, &nh);
                    int count = 0, near_thr = 0;
                    for (int c = 0; c < Cf; c++) top_data[v * Cf + c] = 0;
                    if (top_label) for (int c = 0; c < C; c++) top_label[v * C + c] = 0;
                    for (int x = px - ks; x <= px + ks; x++)
                        for (int y = py - ks; y <= py + ks; y++)
                            if (x >= 0 && x < W && y >= 0 && y < H) {
                                size_t pix = ((size_t)n * H + y) * W + x;
                                float diff = fabsf(depth[pix] - Z1);
                                if (fabsf(diff - threshold) < 1e-5f) near_thr = 1;
                                if (diff < threshold) {
                                    count++;
                                    for (int c = 0; c < Cf; c++) top_data[v * Cf + c] += data[pix * Cf + c];
                                    if (top_label)
                                        for (int c = 0; c < C; c++) top_label[v * C + c] += label[pix * C + c];
                                }
                            }
                    if (ambig) ambig[v] = (unsigned char)(nh || near_thr);
                    if (count == 0) {
                        if (top_flag) for (int c = 0; c < Cf; c++) top_flag[v * Cf + c] = 0;
                        if (top_label) for (int c = 0; c < C; c++) top_label[v * C + c] = label_3d[v * C + c];
                    } else {
                        for (int c = 0; c < Cf; c++) top_data[v * Cf + c] /= count;
                        if (top_flag) for (int c = 0; c < Cf; c++) top_flag[v * Cf + c] = 1;
                        if (top_label) for (int c = 0; c < C; c++) top_label[v * C + c] /= count;
                    }
                }
    return 0;
}

/* the windows of the window average, for test coverage: per voxel the hit count and whether the image border clips the
 * (2 ks + 1)^2 window */
int pcnn_oracle_voxel_window(const float* depth, const float* meta, int B, int H, int W, int num_meta, int G, int ks,
                             float threshold, int* count, unsigned char* clipped)
{
#pragma omp parallel for collapse(2)
    for (int n = 0; n < B; n++)
        for (int d = 0; d < G; d++)
            for (int h = 0; h < G; h++)
                for (int w = 0; w < G; w++) {
                    size_t v = (((size_t)n * G + d) * G + h) * G + w;
                    int px, py, cnt = 0;
                    float Z1;
                    voxel_to_pixel(meta + (size_t)n * num_meta, d, h, w, &px, &py, &Z1, NULL);
                    for (int x = px - ks; x <= px + ks; x++)
                        for (int y = py - ks; y <= py + ks; y++)
                            if (x >= 0 && x < W && y >= 0 && y < H && fabsf(depth[((size_t)n * H + y) * W + x] - Z1) < threshold)
                                cnt++;
                    count[v] = cnt;
                    clipped[v] = (unsigned char)(px - ks < 0 || px + ks > W - 1 || py - ks < 0 || py + ks > H - 1);
                }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* Averagedistance — average_distance_loss/average_distance_loss_op_gpu.cu.cc:34-252 */
/* ------------------------------------------------------------------------- */
static void quat_rot(float s, float u, float v, float w, float* R)
{
    /* .cu.cc:63-71 — un-normalised formula */
    R[0] = s * s + u * u - v * v - w * w; R[1] = 2 * (u * v - s * w); R[2] = 2 * (u * w + s * v);
    R[3] = 2 * (u * v + s * w); R[4] = s * s - u * u + v * v - w * w; R[5] = 2 * (v * w - s * u);
    R[6] = 2 * (u * w - s * v); R[7] = 2 * (v * w + s * u); R[8] = s * s - u * u - v * v + w * w;
}

int pcnn_oracle_average_distance(const float* pred, const float* target, const float* weight, const float* point,
                                 const float* symmetry, int N, int C, int P, float margin, float* loss_out,
                                 float* bottom_diff, int* near_margin_count)
{
    double loss = 0; /* accumulated in double: tolerance rel 1e-4 vs fp32 device sums */
    int near = 0;
    memset(bottom_diff, 0, sizeof(float) * (size_t)N * 4 * C);
    for (int n = 0; n < N; n++) {
        int cls = -1;
        for (int i = 0; i < C; i++)
            if (weight[(size_t)n * 4 * C + 4 * i] > 0) { cls = i; break; }
        if (cls < 0) continue;
        const float* tq = target + (size_t)n * 4 * C + 4 * cls;
        const float* pq = pred + (size_t)n * 4 * C + 4 * cls;
        float Rg[9], Ru[9];
        quat_rot(tq[0], tq[1], tq[2], tq[3], Rg);
        quat_rot(pq[0], pq[1], pq[2], pq[3], Ru);
        float s = pq[0], u = pq[1], v = pq[2], w = pq[3];
        /* derivative matrices .cu.cc:96-139 */
        float D[4][9] = {{2 * s, -2 * w, 2 * v, 2 * w, 2 * s, -2 * u, -2 * v, 2 * u, 2 * s},
                         {2 * u, 2 * v, 2 * w, 2 * v, -2 * u, -2 * s, 2 * w, 2 * s, -2 * u},
                         {-2 * v, 2 * u, 2 * s, 2 * u, 2 * v, 2 * w, -2 * s, 2 * w, -2 * v},
                         {-2 * w, -2 * s, 2 * u, 2 * s, -2 * w, 2 * v, 2 * u, 2 * v, 2 * w}};
        const float* pts = point + (size_t)cls * P * 3;
        double g[4] = {0, 0, 0, 0};
        float* rot2 = (float*)malloc(sizeof(float) * 3 * (size_t)P);
        for (int i = 0; i < P; i++) {
            const float* q = pts + 3 * i;
            rot2[3 * i + 0] = Rg[0] * q[0] + Rg[1] * q[1] + Rg[2] * q[2];
            rot2[3 * i + 1] = Rg[3] * q[0] + Rg[4] * q[1] + Rg[5] * q[2];
            rot2[3 * i + 2] = Rg[6] * q[0] + Rg[7] * q[1] + Rg[8] * q[2];
        }
        for (int p = 0; p < P; p++) {
            const float* q = pts + 3 * p;
            float x1 = Ru[0] * q[0] + Ru[1] * q[1] + Ru[2] * q[2];
            float y1 = Ru[3] * q[0] + Ru[4] * q[1] + Ru[5] * q[2];
            float z1 = Ru[6] * q[0] + Ru[7] * q[1] + Ru[8] * q[2];
            int jmin = p;
            if (symmetry[cls] > 0) {
                float dmin = FLT_MAX;
                for (int i = 0; i < P; i++) {
                    float ex = x1 - rot2[3 * i], ey = y1 - rot2[3 * i + 1], ez = z1 - rot2[3 * i + 2];
                    float dd = ex * ex + ey * ey + ez * ez;
                    if (dd < dmin) { dmin = dd; jmin = i; }
                }
            }
            float ex = x1 - rot2[3 * jmin], ey = y1 - rot2[3 * jmin + 1], ez = z1 - rot2[3 * jmin + 2];
            float dist = ex * ex + ey * ey + ez * ez;
            if (fabsf(dist - margin) < 1e-6f) near++;
            if (dist < margin) continue;
            loss += (double)(dist - margin) / (2.0 * N * P);
            float e[3] = {ex, ey, ez};
            for (int j = 0; j < 3; j++)
                for (int k = 0; k < 3; k++)
                    for (int a = 0; a < 4; a++) g[a] += (double)(e[j] * q[k] * D[a][j * 3 + k] / (float)(N * P));
        }
        for (int a = 0; a < 4; a++) bottom_diff[(size_t)n * 4 * C + 4 * cls + a] = (float)g[a];
        free(rot2);
    }
    *loss_out = (float)loss;
    if (near_margin_count) *near_margin_count = near;
    return 0;
}
