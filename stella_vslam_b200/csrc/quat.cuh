// quat.cuh -- Eigen's quaternion <-> rotation-matrix conversions (fp64), shared by the bundle adjusters (lba_kernels.cu) and the
// Sim3 algebra of the pose-graph optimiser (sim3.cuh).  Quaternions are stored as Eigen's coeffs(): (x, y, z, w); matrices row-major.
#pragma once

#include <cmath>

namespace b200 {

// QuaternionBase::toRotationMatrix
__host__ __device__ inline void quat_to_rot(const double* q, double* R) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
// Quaternion(const Matrix3&): quaternionbase_assign_impl
__host__ __device__ inline void rot_to_quat(const double* R, double* q) {
    double t = R[0] + R[4] + R[8];
    if (t > 0) {
        t = sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (R[7] - R[5]) * t; q[1] = (R[2] - R[6]) * t; q[2] = (R[3] - R[1]) * t;
    } else {
        int i = 0;
        if (R[4] > R[0]) i = 1;
        if (R[8] > R[i * 3 + i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(R[i * 3 + i] - R[j * 3 + j] - R[k * 3 + k] + 1.0);
        double qq[4];
        qq[i] = 0.5 * t;
        t = 0.5 / t;
        qq[3] = (R[k * 3 + j] - R[j * 3 + k]) * t;
        qq[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
        qq[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
        q[0] = qq[0]; q[1] = qq[1]; q[2] = qq[2]; q[3] = qq[3];
    }
}
__host__ __device__ inline void quat_normalize(double* q) {  // SE3Quat::normalizeRotation (also g2o::Sim3::normalizeRotation)
    if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}

}  // namespace b200
