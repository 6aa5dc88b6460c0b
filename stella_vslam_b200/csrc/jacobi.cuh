// jacobi.cuh -- fp64 helpers and the 2x2 step of Eigen::JacobiSVD's two-sided sweeps (real_2x2_jacobi_svd + JacobiRotation::makeJacobi,
// restated from Eigen 3.3/3.4's Jacobi and JacobiSVD modules), shared by the triangulation (triangulate.cuh) and EPnP (epnp.cuh).
//
// Every operation is an explicit round-to-nearest intrinsic, so nothing is contracted whatever the translation unit's -fmad setting.
#pragma once

#include <cfloat>

namespace b200 {
namespace tri {

constexpr int kMaxSweeps = 64;  // a 4x4 or 12x12 converges in a handful of sweeps; hitting the bound is reported, never looped on

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
    return da(da(dm(a0, b0), dm(a1, b1)), dm(a2, b2));
}

// apply_rotation_in_the_plane(x, y, (c, s)) on element k of two vectors
__device__ __forceinline__ void rot2(double& x, double& y, double c, double s) {
    const double xi = x, yi = y;
    x = da(dm(c, xi), dm(s, yi));
    y = da(dm(-s, xi), dm(c, yi));
}

// real_2x2_jacobi_svd on the block (m00 m01; m10 m11) = (W(p,p) W(p,q); W(q,p) W(q,q)): j_left = (cl, sl), j_right = (cr, sr).
// The sweep then applies j_left to rows p, q (and to U's columns p, q as j_left.transpose() on the right) and j_right to columns p, q.
__device__ __forceinline__ void jacobi_2x2(double m00, double m01, double m10, double m11, double& cl, double& sl, double& cr, double& sr) {
    double c1 = 1.0, s1 = 0.0;
    const double t = da(m00, m11), d = ds(m10, m01);
    if (!(fabs(d) < DBL_MIN)) {
        const double u = dd(t, d);
        const double tmp = __dsqrt_rn(da(1.0, dm(u, u)));
        s1 = dd(1.0, tmp);
        c1 = dd(u, tmp);
    }
    if (!(c1 == 1.0 && s1 == 0.0)) {
        rot2(m00, m10, c1, s1);
        rot2(m01, m11, c1, s1);
    }
    // makeJacobi(m00, m01, m11)
    cr = 1.0;
    sr = 0.0;
    const double deno = dm(2.0, fabs(m01));
    if (!(deno < DBL_MIN)) {
        const double tau = dd(ds(m00, m11), deno);
        const double w = __dsqrt_rn(da(dm(tau, tau), 1.0));
        const double tt = tau > 0.0 ? dd(1.0, da(tau, w)) : dd(1.0, ds(tau, w));
        const double sign_t = tt > 0.0 ? 1.0 : -1.0;
        const double n = dd(1.0, __dsqrt_rn(da(dm(tt, tt), 1.0)));
        sr = dm(dm(dm(-sign_t, dd(m01, fabs(m01))), fabs(tt)), n);
        cr = n;
    }
    // j_left = rot1 * j_right^T
    cl = ds(dm(c1, cr), dm(s1, -sr));
    sl = da(dm(c1, -sr), dm(s1, cr));
}

}  // namespace tri
}  // namespace b200
