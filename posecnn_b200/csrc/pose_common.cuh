// pose_common.cuh — rotation helpers shared by the kernels that read or write quaternion pose rows (train_targets.cu: the
// pose blob; coord_pose.cu: the VERTEX_REG_3D detection records; evaluate.cu: the scored estimates; det.cu: the box-fitted
// translations of the detection records).
#pragma once
#include "common.cuh"

namespace pcnn {

// mat2quat is transforms3d's (Bar-Itzhack): eigenvector of the largest eigenvalue of the symmetric 4x4 K matrix, here
// by cyclic Jacobi rotations in double, w made non-negative.
__device__ inline void mat2quat_d(const float* __restrict__ rt /*3x4 row-major*/, float q[4])
{
    // transforms3d: `Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = M.flat` (row-major flat order: Qyx = M[0][1], Qxy = M[1][0], ...)
    const double Qxx = rt[0], Qyx = rt[1], Qzx = rt[2], Qxy = rt[4], Qyy = rt[5], Qzy = rt[6], Qxz = rt[8], Qyz = rt[9], Qzz = rt[10];
    double A[4][4] = {{Qxx - Qyy - Qzz, Qyx + Qxy, Qzx + Qxz, Qyz - Qzy},
                      {Qyx + Qxy, Qyy - Qxx - Qzz, Qzy + Qyz, Qzx - Qxz},
                      {Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, Qxy - Qyx},
                      {Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz}};
    double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) A[i][j] /= 3.0;
    for (int sweep = 0; sweep < 30; sweep++) {
        double off = 0;
        for (int i = 0; i < 4; i++)
            for (int j = i + 1; j < 4; j++) off += A[i][j] * A[i][j];
        if (off < 1e-30) break;
        for (int pI = 0; pI < 3; pI++)
            for (int qI = pI + 1; qI < 4; qI++) {
                if (fabs(A[pI][qI]) < 1e-300) continue;
                const double theta = (A[qI][qI] - A[pI][pI]) / (2.0 * A[pI][qI]);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
                for (int k = 0; k < 4; k++) {
                    const double akp = A[k][pI], akq = A[k][qI];
                    A[k][pI] = c * akp - sn * akq; A[k][qI] = sn * akp + c * akq;
                }
                for (int k = 0; k < 4; k++) {
                    const double apk = A[pI][k], aqk = A[qI][k];
                    A[pI][k] = c * apk - sn * aqk; A[qI][k] = sn * apk + c * aqk;
                }
                for (int k = 0; k < 4; k++) {
                    const double vkp = V[k][pI], vkq = V[k][qI];
                    V[k][pI] = c * vkp - sn * vkq; V[k][qI] = sn * vkp + c * vkq;
                }
            }
    }
    int best = 0;
    for (int k = 1; k < 4; k++)
        if (A[k][k] > A[best][best]) best = k;
    double w = V[3][best], x = V[0][best], y = V[1][best], z = V[2][best];   // vecs[[3, 0, 1, 2], argmax]
    if (w < 0) { w = -w; x = -x; y = -y; z = -z; }
    q[0] = (float)w; q[1] = (float)x; q[2] = (float)y; q[3] = (float)z;
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

}  // namespace pcnn
