// sim3.cuh -- g2o::Sim3 (g2o/types/sim3/sim3.h, upstream tag 20230223_git; not part of the reference tree) and the pose-graph edge
// optimize/internal/sim3/graph_opt_edge.h / shot_vertex.h, restated in fp64 for host and device.
//
// Storage is g2o's: rotation().coeffs() = (x, y, z, w), translation(), scale().  Every expression is evaluated left to right in the
// order written here, and the files including this header are compiled without FMA contraction (build.py): the pose-graph
// Jacobian is a central difference at delta = 1e-9, which amplifies any rounding difference by about 5e8.  tests/pgo_oracle.c
// restates the same functions in the same order.
//
// Lines marked "EXT?" restate upstream g2o / Eigen from its published source where the exact form (not the mathematics) could not
// be checked against the reference tree: Eigen evaluates some of these sums in vectorised order, so they agree with g2o to rounding.
#pragma once

#include <cmath>

#include "quat.cuh"

namespace b200 {
namespace sim3 {

struct Sim3 {
    double q[4];  // x y z w
    double t[3];
    double s;
};

constexpr double kEps = 0.00001;  // sim3.h: "double eps = cst(0.00001)" in the exp constructor and in log()

__host__ __device__ inline void skew(const double* w, double* O) {
    O[0] = 0.0;   O[1] = -w[2]; O[2] = w[1];
    O[3] = w[2];  O[4] = 0.0;   O[5] = -w[0];
    O[6] = -w[1]; O[7] = w[0];  O[8] = 0.0;
}
// 3x3 product, each coefficient ((a0 b0 + a1 b1) + a2 b2)  (EXT? Eigen's lazy-product redux order)
__host__ __device__ inline void mat3_mul(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__host__ __device__ inline void mat3_vec(const double* A, const double* v, double* out) {
    for (int i = 0; i < 3; ++i) out[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
__host__ __device__ inline void cross(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
// QuaternionBase::_transformVector: uv = 2 (q.vec x v); v + w uv + q.vec x uv
__host__ __device__ inline void quat_rotate(const double* q, const double* v, double* out) {
    double uv[3], c[3];
    cross(q, v, uv);
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    cross(q, uv, c);
    for (int i = 0; i < 3; ++i) out[i] = v[i] + q[3] * uv[i] + c[i];
}
// Quaternion product a * b  (EXT? Eigen's scalar quat_product; the SSE2 path for double groups the same four products per term)
__host__ __device__ inline void quat_mul(const double* a, const double* b, double* r) {
    r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
}

// Sim3(const Matrix3& R, const Vector3& t, double s): r(Quaternion(R)), then normalizeRotation()
__host__ __device__ inline Sim3 from_rts(const double* R, const double* t, double s) {
    Sim3 o;
    rot_to_quat(R, o.q);
    quat_normalize(o.q);
    o.t[0] = t[0]; o.t[1] = t[1]; o.t[2] = t[2];
    o.s = s;
    return o;
}

// Sim3::operator*: r = r1 r2, t = s1 (r1 t2) + t1, s = s1 s2 (no normalisation)
__host__ __device__ inline Sim3 mul(const Sim3& a, const Sim3& b) {
    Sim3 o;
    quat_mul(a.q, b.q, o.q);
    double rt[3];
    quat_rotate(a.q, b.t, rt);
    for (int i = 0; i < 3; ++i) o.t[i] = a.s * rt[i] + a.t[i];
    o.s = a.s * b.s;
    return o;
}

// Sim3::inverse(): Sim3(r.conjugate(), r.conjugate() * ((-1. / s) * t), 1. / s), whose constructor normalises the rotation
__host__ __device__ inline Sim3 inverse(const Sim3& a) {
    Sim3 o;
    const double qc[4] = {-a.q[0], -a.q[1], -a.q[2], a.q[3]};
    const double f = -1. / a.s;
    const double st[3] = {f * a.t[0], f * a.t[1], f * a.t[2]};
    quat_rotate(qc, st, o.t);
    o.q[0] = qc[0]; o.q[1] = qc[1]; o.q[2] = qc[2]; o.q[3] = qc[3];
    o.s = 1. / a.s;
    quat_normalize(o.q);
    return o;
}

// Sim3::map: s (r xyz) + t
__host__ __device__ inline void map(const Sim3& a, const double* p, double* out) {
    double rp[3];
    quat_rotate(a.q, p, rp);
    for (int i = 0; i < 3; ++i) out[i] = a.s * rp[i] + a.t[i];
}

// Sim3(const Vector7& update): omega = update[0:3], upsilon = update[3:6], sigma = update[6]
__host__ __device__ inline Sim3 exp7(const double* u) {
    const double omega[3] = {u[0], u[1], u[2]};
    const double ups[3] = {u[3], u[4], u[5]};
    const double sigma = u[6];
    const double theta = sqrt(omega[0] * omega[0] + omega[1] * omega[1] + omega[2] * omega[2]);
    double O[9], O2[9], R[9];
    skew(omega, O);
    Sim3 o;
    o.s = exp(sigma);
    mat3_mul(O, O, O2);
    double A, B, Cc;
    if (fabs(sigma) < kEps) {
        Cc = 1;
        if (theta < kEps) {
            A = 1. / 2.;
            B = 1. / 6.;
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + O[k] + O2[k];  // EXT? g2o writes I + Omega + Omega*Omega
        } else {
            const double theta2 = theta * theta;
            A = (1 - cos(theta)) / (theta2);
            B = (theta - sin(theta)) / (theta2 * theta);
            const double f1 = sin(theta) / theta, f2 = (1 - cos(theta)) / (theta * theta);
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + f1 * O[k] + f2 * O2[k];
        }
    } else {
        Cc = (o.s - 1) / sigma;
        if (theta < kEps) {
            const double sigma2 = sigma * sigma;
            A = ((sigma - 1) * o.s + 1) / sigma2;
            B = ((0.5 * sigma2 - sigma + 1) * o.s - 1) / (sigma2 * sigma);  // the theta -> 0 limit of the general B
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + O[k] + O2[k];  // EXT? as above
        } else {
            const double f1 = sin(theta) / theta, f2 = (1 - cos(theta)) / (theta * theta);
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + f1 * O[k] + f2 * O2[k];
            const double a = o.s * sin(theta);
            const double b = o.s * cos(theta);
            const double theta2 = theta * theta;
            const double sigma2 = sigma * sigma;
            const double c = theta2 + sigma2;
            A = (a * sigma + (1 - b) * theta) / (theta * c);
            B = (Cc - ((b - 1) * sigma + a * theta) / (c)) * 1. / (theta2);
        }
    }
    rot_to_quat(R, o.q);  // r = Quaternion(R): no normalisation in this constructor (EXT?)
    double W[9];
    for (int k = 0; k < 9; ++k) W[k] = A * O[k] + B * O2[k] + ((k % 4 == 0) ? Cc : 0.0);  // A*Omega + B*Omega2 + C*I
    mat3_vec(W, ups, o.t);
    return o;
}

// W.lu().solve(t): Eigen's PartialPivLU (first largest pivot, column scaled by division, rank-1 update), then unit-lower and upper
// substitution  (EXT? Eigen's triangular-solve summation order)
__host__ __device__ inline void lu3_solve(const double* Win, const double* rhs, double* x) {
    double a[9];
    for (int k = 0; k < 9; ++k) a[k] = Win[k];
    int perm[3] = {0, 1, 2};
    for (int k = 0; k < 3; ++k) {
        int p = k;
        double best = fabs(a[3 * k + k]);
        for (int i = k + 1; i < 3; ++i)
            if (fabs(a[3 * i + k]) > best) { best = fabs(a[3 * i + k]); p = i; }
        if (p != k) {
            for (int j = 0; j < 3; ++j) { const double tmp = a[3 * k + j]; a[3 * k + j] = a[3 * p + j]; a[3 * p + j] = tmp; }
            const int tp = perm[k]; perm[k] = perm[p]; perm[p] = tp;
        }
        if (best != 0.0)
            for (int i = k + 1; i < 3; ++i) a[3 * i + k] /= a[3 * k + k];
        for (int i = k + 1; i < 3; ++i)
            for (int j = k + 1; j < 3; ++j) a[3 * i + j] -= a[3 * i + k] * a[3 * k + j];
    }
    double y[3];
    for (int i = 0; i < 3; ++i) {
        double v = rhs[perm[i]];
        for (int j = 0; j < i; ++j) v -= a[3 * i + j] * y[j];
        y[i] = v;
    }
    for (int i = 2; i >= 0; --i) {
        double v = y[i];
        for (int j = i + 1; j < 3; ++j) v -= a[3 * i + j] * x[j];
        x[i] = v / a[3 * i + i];
    }
}

// Sim3::log(): (omega, upsilon, sigma)
__host__ __device__ inline void log7(const Sim3& g, double* res) {
    const double sigma = log(g.s);
    double R[9], omega[3], O[9], O2[9];
    quat_to_rot(g.q, R);
    const double d = 0.5 * (R[0] + R[4] + R[8] - 1);
    const double dR[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};  // deltaR(R)
    double A, B, Cc;
    if (fabs(sigma) < kEps) {
        Cc = 1;
        if (d > 1 - kEps) {
            for (int i = 0; i < 3; ++i) omega[i] = 0.5 * dR[i];
            A = 1. / 2.;
            B = 1. / 6.;
        } else {
            const double theta = acos(d);
            const double theta2 = theta * theta;
            const double f = theta / (2 * sqrt(1 - d * d));
            for (int i = 0; i < 3; ++i) omega[i] = f * dR[i];
            A = (1 - cos(theta)) / (theta2);
            B = (theta - sin(theta)) / (theta2 * theta);
        }
    } else {
        Cc = (g.s - 1) / sigma;
        if (d > 1 - kEps) {
            const double sigma2 = sigma * sigma;
            for (int i = 0; i < 3; ++i) omega[i] = 0.5 * dR[i];
            A = ((sigma - 1) * g.s + 1) / (sigma2);
            B = ((0.5 * sigma2 - sigma + 1) * g.s - 1) / (sigma2 * sigma);
        } else {
            const double theta = acos(d);
            const double f = theta / (2 * sqrt(1 - d * d));
            for (int i = 0; i < 3; ++i) omega[i] = f * dR[i];
            const double theta2 = theta * theta;
            const double a = g.s * sin(theta);
            const double b = g.s * cos(theta);
            const double c = theta2 + sigma * sigma;
            A = (a * sigma + (1 - b) * theta) / (theta * c);
            B = (Cc - ((b - 1) * sigma + a * theta) / (c)) * 1. / (theta2);
        }
    }
    skew(omega, O);
    mat3_mul(O, O, O2);
    double W[9];
    for (int k = 0; k < 9; ++k) W[k] = A * O[k] + B * O2[k] + ((k % 4 == 0) ? Cc : 0.0);
    double ups[3];
    lu3_solve(W, g.t, ups);
    res[0] = omega[0]; res[1] = omega[1]; res[2] = omega[2];
    res[3] = ups[0]; res[4] = ups[1]; res[5] = ups[2];
    res[6] = sigma;
}

// Host-side input check of the optimisers: finite, scale > 0, and a quaternion near unit norm (a zero or denormal one would divide
// by ~0 in inverse()'s normalisation).
inline bool well_formed(const double* q, const double* t, double s) {
    for (int k = 0; k < 4; ++k)
        if (!std::isfinite(q[k])) return false;
    for (int k = 0; k < 3; ++k)
        if (!std::isfinite(t[k])) return false;
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    return std::isfinite(s) && s > 0 && n2 > 0.25 && n2 < 4.0;
}

// shot_vertex::oplusImpl and transform_vertex::oplusImpl: estimate <- Sim3(update) * estimate, update(6) zeroed under fix_scale
__host__ __device__ inline Sim3 oplus(const Sim3& est, const double* upd, bool fix_scale) {
    double u[7] = {upd[0], upd[1], upd[2], upd[3], upd[4], upd[5], fix_scale ? 0.0 : upd[6]};
    return mul(exp7(u), est);
}

// graph_opt_edge::computeError: log(C * v1 * v2^-1)
__host__ __device__ inline void edge_error(const Sim3& meas, const Sim3& v1, const Sim3& v2, double* e) {
    const Sim3 c1 = mul(meas, v1);
    log7(mul(c1, inverse(v2)), e);
}

}  // namespace sim3
}  // namespace b200
