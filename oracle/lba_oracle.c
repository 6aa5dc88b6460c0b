/*
 * oracle/lba_oracle.c -- TEST INFRASTRUCTURE (see oracle.h).  CPU restatement of optimize::local_bundle_adjuster_g2o.
 *
 * PARITY UNPINNED: the reference solves local BA through g2o (tag 20230223_git) + Eigen 3.3.7, neither of which is in
 * the reference tree nor a dependency of this repository, and the reference ships no test or golden vector for this path (SURVEY.md 8c).
 * This file restates (a) the reference's own code -- the optimisation protocol of
 * optimize/local_bundle_adjuster_g2o.cc:149-375, the residuals/Jacobians of optimize/internal/se3/
 * {perspective,equirectangular}_reproj_edge.h, reproj_edge_wrapper.h, shot_vertex.h, landmark_vertex.h,
 * terminate_action.cc -- and (b) g2o's published algorithm: BaseBinaryEdge::constructQuadraticForm with
 * RobustKernelHuber, BlockSolver_6_3 Schur complement, OptimizationAlgorithmLevenberg (tau 1e-5, rho/scale rule,
 * <= 10 trials), SparseOptimizer::optimize loop, SE3Quat::exp.  tests/test_lba_cpu.py checks it against an independent
 * dense numpy Gauss-Newton step and numerical Jacobians on small problems.  Since round 2 the OPTIMUM it reaches is pinned:
 * tests/test_lba_scipy.py minimises the same Huber cost over the same edges with scipy.optimize.least_squares (mono / stereo /
 * equirectangular windows) and compares chi2, outlier set and the optimum itself; what stays unpinned is the LM PATH (iteration
 * counts, lambda schedule, the terminate action), which only g2o itself could confirm.  The CUDA path is held to 1e-5 relative
 * against this file.  orc_global_ba_solve (optimize/global_bundle_adjuster.cc) is one round of the same machinery.
 * orc_pose_optimize (optimize/pose_optimizer_g2o.cc:38-175, SURVEY 8f N1) reuses the same edge and LM code with one free pose and
 * fixed landmarks: equally unpinned (tests/test_pose_opt_cpu.py: protocol properties and ground truth on synthetic frames).
 */
#define _GNU_SOURCE
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

/* ---------- small dense helpers (row-major) ---------- */
static void quat_to_rot(const double* q, double* R) { /* q = (x,y,z,w), Eigen toRotationMatrix */
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
static void rot_to_quat(const double* R, double* q) { /* Eigen Quaternion(Matrix3) */
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
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (R[k * 3 + j] - R[j * 3 + k]) * t;
        q[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
        q[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
    }
}
static void quat_normalize(double* q) { /* SE3Quat::normalizeRotation */
    if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
static void quat_mul(const double* a, const double* b, double* r) { /* r = a * b */
    r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
}
static void quat_rotate(const double* q, const double* v, double* r) { /* Eigen: v + w*uv + q.vec x uv, uv = 2 q.vec x v */
    double uv[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    r[0] = v[0] + q[3] * uv[0] + (q[1] * uv[2] - q[2] * uv[1]);
    r[1] = v[1] + q[3] * uv[1] + (q[2] * uv[0] - q[0] * uv[2]);
    r[2] = v[2] + q[3] * uv[2] + (q[0] * uv[1] - q[1] * uv[0]);
}
/* shot_vertex::oplusImpl (shot_vertex.h:55-58): estimate <- SE3Quat::exp(update) * estimate, update = [omega, upsilon] */
static void se3_oplus(double* q, double* t, const double* upd) {
    const double* om = upd;
    const double* up = upd + 3;
    const double theta = sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
    const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
    double O2[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O2[i * 3 + j] = O[i * 3] * O[j] + O[i * 3 + 1] * O[3 + j] + O[i * 3 + 2] * O[6 + j];
    double a, b, c, d;
    if (theta < 0.00001) {
        a = 1.0; b = 0.5; c = 0.5; d = 1.0 / 6.0;
    } else {
        a = sin(theta) / theta;
        b = (1 - cos(theta)) / (theta * theta);
        c = b;
        d = (theta - sin(theta)) / (theta * theta * theta);
    }
    double R[9], V[9];
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1.0 : 0.0;
        R[i] = I + a * O[i] + b * O2[i];
        V[i] = I + c * O[i] + d * O2[i];
    }
    double dq[4], dt[3];
    rot_to_quat(R, dq);
    quat_normalize(dq);
    for (int i = 0; i < 3; ++i) dt[i] = V[i * 3] * up[0] + V[i * 3 + 1] * up[1] + V[i * 3 + 2] * up[2];
    /* (dq,dt) * (q,t): t' = dt + dq*t ; q' = dq*q */
    double rt[3], nq[4];
    quat_rotate(dq, t, rt);
    t[0] = dt[0] + rt[0]; t[1] = dt[1] + rt[1]; t[2] = dt[2] + rt[2];
    quat_mul(dq, q, nq);
    quat_normalize(nq);
    memcpy(q, nq, sizeof(nq));
}

/* ---------- problem state ---------- */
typedef struct {
    const orc_lba_problem_t* P;
    double* q;      /* K x 4 */
    double* t;      /* K x 3 */
    double* pts;    /* L x 3 */
    int* pose_col;  /* K: index among free poses or -1 */
    int* pt_col;    /* L: index among free points or -1 */
    int nfp, nfl;
    uint8_t* level;  /* E: 0 active, 1 outlier */
    uint8_t* robust; /* E: Huber on/off (dropped before the second round) */
    double* err;     /* E x 3 last computed error (only refreshed while the edge is active) */
    /* system */
    double *Hpp, *bp; /* nfp x 36, nfp x 6 (diagonal blocks) */
    double *Hll, *bl; /* nfl x 9, nfl x 3 */
    double* Hpl;      /* E x 18 (6x3 per edge, valid if both free) */
    double *xp, *xl;
} lba_t;

static int edge_dim(const orc_lba_problem_t* P, int e) { return P->e_obs[3 * e + 2] < 0 ? 2 : 3; } /* is_monocular_ = x_right < 0 */

/* computeError of the three edge types (perspective_reproj_edge.h:67-72,118-120,175-180,236-239; equirectangular_reproj_edge.h:64-69,130-134) */
static void edge_error(const lba_t* S, int e, double* err, double* pc_out) {
    const orc_lba_problem_t* P = S->P;
    const int ip = P->e_pose[e], il = P->e_point[e];
    const orc_camera_t* c = &P->cams[P->e_cam[e]];
    double pc[3];
    quat_rotate(S->q + 4 * ip, S->pts + 3 * il, pc);
    pc[0] += S->t[3 * ip]; pc[1] += S->t[3 * ip + 1]; pc[2] += S->t[3 * ip + 2];
    const double ox = P->e_obs[3 * e], oy = P->e_obs[3 * e + 1], orr = P->e_obs[3 * e + 2];
    if (c->model == 1) { /* equirectangular */
        const double theta = atan2(pc[0], pc[2]);
        const double phi = -asin(pc[1] / sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]));
        err[0] = ox - c->cols * (0.5 + theta / (2 * M_PI));
        err[1] = oy - c->rows * (0.5 - phi / M_PI);
        err[2] = 0;
    } else {
        const double rx = c->fx * pc[0] / pc[2] + c->cx;
        err[0] = ox - rx;
        err[1] = oy - (c->fy * pc[1] / pc[2] + c->cy);
        err[2] = (orr < 0) ? 0 : orr - (rx - c->fxb / pc[2]);
    }
    if (pc_out) memcpy(pc_out, pc, sizeof(pc));
}

/* linearizeOplus: Ji (dim x 3, landmark) and Jj (dim x 6, pose; rotation first) */
static void edge_jacobians(const lba_t* S, int e, double* Ji, double* Jj) {
    const orc_lba_problem_t* P = S->P;
    const int ip = P->e_pose[e], il = P->e_point[e];
    const orc_camera_t* c = &P->cams[P->e_cam[e]];
    double pc[3], R[9];
    quat_rotate(S->q + 4 * ip, S->pts + 3 * il, pc);
    pc[0] += S->t[3 * ip]; pc[1] += S->t[3 * ip + 1]; pc[2] += S->t[3 * ip + 2];
    quat_to_rot(S->q + 4 * ip, R);
    const double x = pc[0], y = pc[1], z = pc[2];
    memset(Ji, 0, sizeof(double) * 9);
    memset(Jj, 0, sizeof(double) * 18);
    if (c->model == 1) { /* equirectangular_reproj_edge.h:71-128 */
        const double L = sqrt(x * x + y * y + z * z);
        double dx[9] = {0, z, -y, 1, 0, 0, R[0], R[1], R[2]};  /* d pcx / d [r, t, pw] */
        double dy[9] = {-z, 0, x, 0, 1, 0, R[3], R[4], R[5]};
        double dz[9] = {y, -x, 0, 0, 0, 1, R[6], R[7], R[8]};
        const double k0 = -(c->cols / (2 * M_PI)) * (1.0 / (x * x + z * z));
        const double k1 = -(c->rows / M_PI) * (1.0 / (L * sqrt(x * x + z * z)));
        for (int j = 0; j < 9; ++j) {
            const double dL = (1.0 / L) * (x * dx[j] + y * dy[j] + z * dz[j]);
            const double j0 = k0 * (z * dx[j] - x * dz[j]);
            const double j1 = k1 * (L * dy[j] - y * dL);
            if (j < 6) { Jj[j] = j0; Jj[6 + j] = j1; } else { Ji[j - 6] = j0; Ji[3 + j - 6] = j1; }
        }
        return;
    }
    const double fx = c->fx, fy = c->fy, z_sq = z * z;
    for (int j = 0; j < 3; ++j) { /* perspective_reproj_edge.h:89-95 */
        Ji[j] = -fx * R[j] / z + fx * x * R[6 + j] / z_sq;
        Ji[3 + j] = -fy * R[3 + j] / z + fy * y * R[6 + j] / z_sq;
    }
    Jj[0] = x * y / z_sq * fx; Jj[1] = -(1.0 + (x * x / z_sq)) * fx; Jj[2] = y / z * fx;
    Jj[3] = -1.0 / z * fx;     Jj[4] = 0.0;                            Jj[5] = x / z_sq * fx;
    Jj[6] = (1.0 + y * y / z_sq) * fy; Jj[7] = -x * y / z_sq * fy; Jj[8] = -x / z * fy;
    Jj[9] = 0.0;                       Jj[10] = -1.0 / z * fy;     Jj[11] = y / z_sq * fy;
    if (P->e_obs[3 * e + 2] >= 0) { /* stereo rows (perspective_reproj_edge.h:203-205,221-226) */
        const double fxb = c->fxb;
        for (int j = 0; j < 3; ++j) Ji[6 + j] = Ji[j] - fxb * R[6 + j] / z_sq;
        Jj[12] = Jj[0] - fxb * y / z_sq; Jj[13] = Jj[1] + fxb * x / z_sq; Jj[14] = Jj[2];
        Jj[15] = Jj[3];                  Jj[16] = 0;                      Jj[17] = Jj[5] - fxb / z_sq;
    }
}

static int depth_is_positive(const lba_t* S, int e) { /* reproj_edge_wrapper.h:233-268 */
    const orc_lba_problem_t* P = S->P;
    if (P->cams[P->e_cam[e]].model == 1) return 1;
    double pc[3];
    const int ip = P->e_pose[e];
    quat_rotate(S->q + 4 * ip, S->pts + 3 * P->e_point[e], pc);
    return 0.0 < pc[2] + S->t[3 * ip + 2];
}

static double edge_chi2(const lba_t* S, int e) { /* e^T (I * inv_sigma_sq) e */
    const double w = (double)S->P->e_inv_sigma_sq[e];
    const double* r = S->err + 3 * e;
    return w * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
}

/* computeActiveErrors + activeRobustChi2 (RobustKernelHuber::robustify rho[0]) */
static double compute_active_errors(lba_t* S) {
    const orc_lba_problem_t* P = S->P;
    double chi = 0;
    for (int e = 0; e < P->n_edges; ++e) {
        if (S->level[e]) continue;
        edge_error(S, e, S->err + 3 * e, NULL);
        const double e2 = edge_chi2(S, e);
        if (S->robust[e]) {
            const double delta = (double)P->e_delta[e], dsqr = delta * delta;
            chi += (e2 <= dsqr) ? e2 : 2 * sqrt(e2) * delta - dsqr;
        } else {
            chi += e2;
        }
    }
    return chi;
}

/* BlockSolver::buildSystem: constructQuadraticForm per active edge */
static void build_system(lba_t* S) {
    const orc_lba_problem_t* P = S->P;
    memset(S->Hpp, 0, sizeof(double) * 36 * (S->nfp ? S->nfp : 1));
    memset(S->bp, 0, sizeof(double) * 6 * (S->nfp ? S->nfp : 1));
    memset(S->Hll, 0, sizeof(double) * 9 * (S->nfl ? S->nfl : 1));
    memset(S->bl, 0, sizeof(double) * 3 * (S->nfl ? S->nfl : 1));
    for (int e = 0; e < P->n_edges; ++e) {
        if (S->level[e]) continue;
        const int cp = S->pose_col[P->e_pose[e]], cl = S->pt_col[P->e_point[e]];
        if (cp < 0 && cl < 0) continue;
        double Ji[9], Jj[18];
        edge_jacobians(S, e, Ji, Jj);
        const int dim = edge_dim(P, e);
        double w = (double)P->e_inv_sigma_sq[e];
        const double* r = S->err + 3 * e;
        double rho1 = 1.0;
        if (S->robust[e]) {
            const double e2 = edge_chi2(S, e), delta = (double)P->e_delta[e];
            if (e2 > delta * delta) rho1 = delta / sqrt(e2);
        }
        const double ww = w * rho1; /* weightedOmega = rho[1] * Omega; omega_r = -Omega e * rho[1] */
        if (cl >= 0) {
            double* H = S->Hll + 9 * cl;
            double* b = S->bl + 3 * cl;
            for (int a = 0; a < 3; ++a) {
                for (int d = 0; d < dim; ++d) b[a] += Ji[d * 3 + a] * (-ww * r[d]);
                for (int c = 0; c < 3; ++c)
                    for (int d = 0; d < dim; ++d) H[a * 3 + c] += Ji[d * 3 + a] * ww * Ji[d * 3 + c];
            }
        }
        if (cp >= 0) {
            double* H = S->Hpp + 36 * cp;
            double* b = S->bp + 6 * cp;
            for (int a = 0; a < 6; ++a) {
                for (int d = 0; d < dim; ++d) b[a] += Jj[d * 6 + a] * (-ww * r[d]);
                for (int c = 0; c < 6; ++c)
                    for (int d = 0; d < dim; ++d) H[a * 6 + c] += Jj[d * 6 + a] * ww * Jj[d * 6 + c];
            }
        }
        if (cp >= 0 && cl >= 0) {
            double* H = S->Hpl + 18 * e; /* 6x3 = Jj^T W Ji */
            for (int a = 0; a < 6; ++a)
                for (int c = 0; c < 3; ++c) {
                    double s = 0;
                    for (int d = 0; d < dim; ++d) s += Jj[d * 6 + a] * ww * Ji[d * 3 + c];
                    H[a * 3 + c] = s;
                }
        }
    }
}

static int inv3(const double* A, double* B) {
    const double c0 = A[4] * A[8] - A[5] * A[7], c1 = A[5] * A[6] - A[3] * A[8], c2 = A[3] * A[7] - A[4] * A[6];
    const double det = A[0] * c0 + A[1] * c1 + A[2] * c2;
    if (det == 0 || !isfinite(det)) return 0;
    const double id = 1.0 / det;
    B[0] = c0 * id; B[1] = (A[2] * A[7] - A[1] * A[8]) * id; B[2] = (A[1] * A[5] - A[2] * A[4]) * id;
    B[3] = c1 * id; B[4] = (A[0] * A[8] - A[2] * A[6]) * id; B[5] = (A[2] * A[3] - A[0] * A[5]) * id;
    B[6] = c2 * id; B[7] = (A[1] * A[6] - A[0] * A[7]) * id; B[8] = (A[0] * A[4] - A[1] * A[3]) * id;
    return 1;
}

/* dense Cholesky solve of the reduced pose system (stands in for g2o::LinearSolverEigen; any exact SPD solve agrees to 1e-5) */
static int chol_solve(double* A, double* b, int n) {
    for (int j = 0; j < n; ++j) {
        double d = A[j * n + j];
        for (int k = 0; k < j; ++k) d -= A[j * n + k] * A[j * n + k];
        if (!(d > 0) || !isfinite(d)) return 0;
        d = sqrt(d);
        A[j * n + j] = d;
        for (int i = j + 1; i < n; ++i) {
            double s = A[i * n + j];
            for (int k = 0; k < j; ++k) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / d;
        }
    }
    for (int i = 0; i < n; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= A[i * n + k] * b[k];
        b[i] = s / A[i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
        double s = b[i];
        for (int k = i + 1; k < n; ++k) s -= A[k * n + i] * b[k];
        b[i] = s / A[i * n + i];
    }
    return 1;
}

/* BlockSolver::solve with Schur complement, lambda added to every diagonal entry of Hpp and Hll */
static int solve_system(lba_t* S, double lambda) {
    const orc_lba_problem_t* P = S->P;
    const int n = 6 * S->nfp;
    double* Hs = (double*)calloc((size_t)(n ? n : 1) * (n ? n : 1), sizeof(double));
    double* bs = (double*)calloc(n ? n : 1, sizeof(double));
    double* Dinv = (double*)malloc(sizeof(double) * 9 * (S->nfl ? S->nfl : 1));
    int ok = 1;
    for (int p = 0; p < S->nfp; ++p) {
        for (int a = 0; a < 6; ++a) {
            for (int c = 0; c < 6; ++c) Hs[(6 * p + a) * n + 6 * p + c] = S->Hpp[36 * p + a * 6 + c];
            Hs[(6 * p + a) * n + 6 * p + a] += lambda;
            bs[6 * p + a] = S->bp[6 * p + a];
        }
    }
    for (int l = 0; l < S->nfl; ++l) {
        double D[9];
        memcpy(D, S->Hll + 9 * l, sizeof(D));
        D[0] += lambda; D[4] += lambda; D[8] += lambda;
        if (!inv3(D, Dinv + 9 * l)) ok = 0;
    }
    /* per-landmark edge lists */
    int* head = (int*)malloc(sizeof(int) * (S->nfl + 1));
    int* list = (int*)malloc(sizeof(int) * (P->n_edges ? P->n_edges : 1));
    memset(head, 0, sizeof(int) * (S->nfl + 1));
    for (int e = 0; e < P->n_edges; ++e) {
        const int cl = S->pt_col[P->e_point[e]];
        if (!S->level[e] && cl >= 0 && S->pose_col[P->e_pose[e]] >= 0) head[cl + 1]++;
    }
    for (int l = 0; l < S->nfl; ++l) head[l + 1] += head[l];
    int* fill = (int*)malloc(sizeof(int) * (S->nfl ? S->nfl : 1));
    memcpy(fill, head, sizeof(int) * S->nfl);
    for (int e = 0; e < P->n_edges; ++e) {
        const int cl = S->pt_col[P->e_point[e]];
        if (!S->level[e] && cl >= 0 && S->pose_col[P->e_pose[e]] >= 0) list[fill[cl]++] = e;
    }
    for (int l = 0; l < S->nfl && ok; ++l) {
        const double* Di = Dinv + 9 * l;
        const double* bl = S->bl + 3 * l;
        for (int a = head[l]; a < head[l + 1]; ++a) {
            const int e1 = list[a], p1 = S->pose_col[P->e_pose[e1]];
            double BD[18]; /* Hpl(e1) * Dinv, 6x3 */
            const double* B1 = S->Hpl + 18 * e1;
            for (int i = 0; i < 6; ++i)
                for (int j = 0; j < 3; ++j) BD[i * 3 + j] = B1[i * 3] * Di[j] + B1[i * 3 + 1] * Di[3 + j] + B1[i * 3 + 2] * Di[6 + j];
            for (int i = 0; i < 6; ++i) bs[6 * p1 + i] -= BD[i * 3] * bl[0] + BD[i * 3 + 1] * bl[1] + BD[i * 3 + 2] * bl[2];
            for (int c = head[l]; c < head[l + 1]; ++c) {
                const int e2 = list[c], p2 = S->pose_col[P->e_pose[e2]];
                const double* B2 = S->Hpl + 18 * e2;
                for (int i = 0; i < 6; ++i)
                    for (int j = 0; j < 6; ++j)
                        Hs[(6 * p1 + i) * n + 6 * p2 + j] -= BD[i * 3] * B2[j * 3] + BD[i * 3 + 1] * B2[j * 3 + 1] + BD[i * 3 + 2] * B2[j * 3 + 2];
            }
        }
    }
    if (ok && n > 0) ok = chol_solve(Hs, bs, n);
    if (ok) {
        memcpy(S->xp, bs, sizeof(double) * n);
        for (int l = 0; l < S->nfl; ++l) {
            double c[3] = {S->bl[3 * l], S->bl[3 * l + 1], S->bl[3 * l + 2]};
            for (int a = head[l]; a < head[l + 1]; ++a) {
                const int e = list[a], p = S->pose_col[P->e_pose[e]];
                const double* B = S->Hpl + 18 * e;
                for (int j = 0; j < 3; ++j)
                    for (int i = 0; i < 6; ++i) c[j] -= B[i * 3 + j] * S->xp[6 * p + i];
            }
            const double* Di = Dinv + 9 * l;
            for (int j = 0; j < 3; ++j) S->xl[3 * l + j] = Di[j * 3] * c[0] + Di[j * 3 + 1] * c[1] + Di[j * 3 + 2] * c[2];
        }
    }
    free(Hs); free(bs); free(Dinv); free(head); free(list); free(fill);
    return ok;
}

static void apply_update(lba_t* S) {
    const orc_lba_problem_t* P = S->P;
    for (int k = 0; k < P->n_poses; ++k)
        if (S->pose_col[k] >= 0) se3_oplus(S->q + 4 * k, S->t + 3 * k, S->xp + 6 * S->pose_col[k]);
    for (int l = 0; l < P->n_points; ++l)
        if (S->pt_col[l] >= 0)
            for (int j = 0; j < 3; ++j) S->pts[3 * l + j] += S->xl[3 * S->pt_col[l] + j]; /* landmark_vertex.h:50-53 */
}

/* SparseOptimizer::optimize(n) with OptimizationAlgorithmLevenberg + terminate_action (terminate_action.cc:36-76).
 * Returns the number of iterations run. */
static double g_gain_thr = 1e-3; /* terminate_action::setGainThreshold; 1e-3 everywhere except optimize_for_initialization */
static int optimize_rounds(lba_t* S, int iterations, volatile uint8_t* stop, orc_lba_stats_t* st, int round) {
    const orc_lba_problem_t* P = S->P;
    uint8_t aux_stop = 0;
    volatile uint8_t* flag = stop ? stop : &aux_stop;
    *flag = 0; /* terminate_action at iteration -1: "let the optimizer run for at least one iteration": reset the stop flag */
    double lambda = 0, ni = 2, last_chi = 0;
    const int K = P->n_poses, L = P->n_points;
    double* bq = (double*)malloc(sizeof(double) * 4 * K);
    double* bt = (double*)malloc(sizeof(double) * 3 * K);
    double* bpts = (double*)malloc(sizeof(double) * 3 * L);
    int it = 0;
    int ok = 1;
    for (; it < iterations && !*flag && ok; ++it) {
        double current_chi = compute_active_errors(S);
        double temp_chi = current_chi;
        build_system(S);
        if (it == 0) { /* computeLambdaInit: tau * max |H_jj| over all free vertices */
            double mx = 0;
            for (int p = 0; p < S->nfp; ++p)
                for (int a = 0; a < 6; ++a) mx = fmax(mx, fabs(S->Hpp[36 * p + a * 7]));
            for (int l = 0; l < S->nfl; ++l)
                for (int a = 0; a < 3; ++a) mx = fmax(mx, fabs(S->Hll[9 * l + a * 4]));
            lambda = 1e-5 * mx;
            ni = 2;
            if (round == 0 && st) st->lambda_init = lambda;
        }
        double rho = 0;
        int qmax = 0;
        do {
            memcpy(bq, S->q, sizeof(double) * 4 * K); /* push */
            memcpy(bt, S->t, sizeof(double) * 3 * K);
            memcpy(bpts, S->pts, sizeof(double) * 3 * L);
            const int ok2 = solve_system(S, lambda);
            if (ok2) apply_update(S);
            temp_chi = compute_active_errors(S);
            if (!ok2) temp_chi = 1.7976931348623157e308;
            rho = current_chi - temp_chi;
            double scale = 0; /* computeScale */
            if (ok2) {
                for (int j = 0; j < 6 * S->nfp; ++j) scale += S->xp[j] * (lambda * S->xp[j] + S->bp[j]);
                for (int j = 0; j < 3 * S->nfl; ++j) scale += S->xl[j] * (lambda * S->xl[j] + S->bl[j]);
            }
            scale += 1e-3;
            rho /= scale;
            if (rho > 0 && isfinite(temp_chi) && ok2) {
                double alpha = 1. - pow((2 * rho - 1), 3);
                alpha = fmin(alpha, 2. / 3.);
                const double sf = fmax(1. / 3., alpha);
                lambda *= sf;
                ni = 2;
                current_chi = temp_chi;
            } else {
                lambda *= ni;
                ni *= 2;
                memcpy(S->q, bq, sizeof(double) * 4 * K); /* pop */
                memcpy(S->t, bt, sizeof(double) * 3 * K);
                memcpy(S->pts, bpts, sizeof(double) * 3 * L);
                if (!isfinite(lambda)) break;
            }
            qmax++;
        } while (rho < 0 && qmax < 10 && !*flag);
        if (qmax == 10 || rho == 0 || !isfinite(lambda)) ok = 0; /* SolverResult::Terminate */
        /* postIteration(it): terminate_action */
        const double chi = compute_active_errors(S);
        if (it == 0) {
            last_chi = chi;
        } else {
            const double gain = (last_chi - chi) / chi;
            last_chi = chi;
            if (gain >= 0 && gain < g_gain_thr) *flag = 1; /* setOptimizerStopFlag: writes the caller's force-stop flag */
        }
        if (st) {
            st->chi2[round] = chi;
            st->lambda_final[round] = lambda;
        }
    }
    free(bq); free(bt); free(bpts);
    if (it == 0 && st) st->chi2[round] = compute_active_errors(S);
    return it;
}

static void state_init(lba_t* Sp, const orc_lba_problem_t* P) {
#define S (*Sp)
    memset(&S, 0, sizeof(S));
    S.P = P;
    const int K = P->n_poses, L = P->n_points, E = P->n_edges;
    S.q = (double*)malloc(sizeof(double) * 4 * (K ? K : 1));
    S.t = (double*)malloc(sizeof(double) * 3 * (K ? K : 1));
    S.pts = (double*)malloc(sizeof(double) * 3 * (L ? L : 1));
    S.pose_col = (int*)malloc(sizeof(int) * (K ? K : 1));
    S.pt_col = (int*)malloc(sizeof(int) * (L ? L : 1));
    for (int k = 0; k < K; ++k) { /* util::converter::to_g2o_SE3 (util/converter.cc:17-21) */
        const double* M = P->pose_cw + 16 * k;
        const double R[9] = {M[0], M[1], M[2], M[4], M[5], M[6], M[8], M[9], M[10]};
        rot_to_quat(R, S.q + 4 * k);
        quat_normalize(S.q + 4 * k);
        S.t[3 * k] = M[3]; S.t[3 * k + 1] = M[7]; S.t[3 * k + 2] = M[11];
        S.pose_col[k] = P->pose_fixed[k] ? -1 : S.nfp++;
    }
    memcpy(S.pts, P->points, sizeof(double) * 3 * L);
    for (int l = 0; l < L; ++l) S.pt_col[l] = (P->point_fixed && P->point_fixed[l]) ? -1 : S.nfl++;
    S.level = (uint8_t*)calloc(E ? E : 1, 1);
    S.robust = (uint8_t*)malloc(E ? E : 1);
    for (int e = 0; e < E; ++e) S.robust[e] = P->e_robust ? P->e_robust[e] : 1;
    S.err = (double*)calloc(3 * (size_t)(E ? E : 1), sizeof(double));
    S.Hpp = (double*)malloc(sizeof(double) * 36 * (S.nfp ? S.nfp : 1));
    S.bp = (double*)malloc(sizeof(double) * 6 * (S.nfp ? S.nfp : 1));
    S.Hll = (double*)malloc(sizeof(double) * 9 * (S.nfl ? S.nfl : 1));
    S.bl = (double*)malloc(sizeof(double) * 3 * (S.nfl ? S.nfl : 1));
    S.Hpl = (double*)calloc(18 * (size_t)(E ? E : 1), sizeof(double));
    S.xp = (double*)calloc(6 * (size_t)(S.nfp ? S.nfp : 1), sizeof(double));
    S.xl = (double*)calloc(3 * (size_t)(S.nfl ? S.nfl : 1), sizeof(double));
#undef S
}
static void state_free(lba_t* S) {
    free(S->q); free(S->t); free(S->pts); free(S->pose_col); free(S->pt_col); free(S->level); free(S->robust); free(S->err);
    free(S->Hpp); free(S->bp); free(S->Hll); free(S->bl); free(S->Hpl); free(S->xp); free(S->xl);
}
static void pose_to_mat(const lba_t* S, int k, double* M) { /* util::converter::to_eigen_mat(SE3Quat) */
    double R[9];
    quat_to_rot(S->q + 4 * k, R);
    M[0] = R[0]; M[1] = R[1]; M[2] = R[2]; M[3] = S->t[3 * k];
    M[4] = R[3]; M[5] = R[4]; M[6] = R[5]; M[7] = S->t[3 * k + 1];
    M[8] = R[6]; M[9] = R[7]; M[10] = R[8]; M[11] = S->t[3 * k + 2];
    M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
}

int orc_lba_solve(const orc_lba_problem_t* P, int iters1, int iters2, volatile uint8_t* force_stop, double* pose_cw_out,
                  double* points_out, uint8_t* outlier_out, orc_lba_stats_t* stats) {
    /* local_bundle_adjuster_g2o.cc:308-310 */
    if (force_stop && *force_stop) return 1;
    lba_t S;
    state_init(&S, P);
    const int K = P->n_poses, L = P->n_points, E = P->n_edges;
    if (stats) memset(stats, 0, sizeof(*stats));

    /* 5. first optimisation (:312-313) */
    const int n1 = optimize_rounds(&S, iters1, force_stop, stats, 0);
    if (stats) stats->iterations[0] = n1;
    /* 6. outliers + second optimisation (:317-348) */
    int run_robust = 1;
    if (force_stop && *force_stop) run_robust = 0;
    if (run_robust) {
        for (int e = 0; e < E; ++e) {
            if (P->e_can_be_outlier && !P->e_can_be_outlier[e]) continue; /* marker edges are not in reproj_edge_wraps */
            const double thr = (edge_dim(P, e) == 2) ? (double)5.99146f : (double)7.81473f; /* constexpr float chi_sq_2D / 3D */
            if (thr < edge_chi2(&S, e) || !depth_is_positive(&S, e)) S.level[e] = 1;
            S.robust[e] = 0;
        }
        const int n2 = optimize_rounds(&S, iters2, force_stop, stats, 1);
        if (stats) stats->iterations[1] = n2;
    }
    /* 7. outlier observations (:354-375): chi2() is the value from the last time the edge was active */
    int n_out = 0;
    for (int e = 0; e < E; ++e) {
        uint8_t o = 0;
        if (!P->e_can_be_outlier || P->e_can_be_outlier[e]) {
            const double thr = (edge_dim(P, e) == 2) ? (double)5.99146f : (double)7.81473f;
            o = (thr < edge_chi2(&S, e) || !depth_is_positive(&S, e)) ? 1 : 0;
        }
        if (outlier_out) outlier_out[e] = o;
        n_out += o;
    }
    if (stats) stats->n_outliers = n_out;
    /* 8. write-back (:393-409): to_eigen_mat(SE3Quat) */
    for (int k = 0; k < K; ++k) {
        double* M = pose_cw_out + 16 * k;
        if (P->pose_fixed[k]) {
            memcpy(M, P->pose_cw + 16 * k, sizeof(double) * 16);
            continue;
        }
        double R[9];
        quat_to_rot(S.q + 4 * k, R);
        M[0] = R[0]; M[1] = R[1]; M[2] = R[2]; M[3] = S.t[3 * k];
        M[4] = R[3]; M[5] = R[4]; M[6] = R[5]; M[7] = S.t[3 * k + 1];
        M[8] = R[6]; M[9] = R[7]; M[10] = R[8]; M[11] = S.t[3 * k + 2];
        M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
    }
    memcpy(points_out, S.pts, sizeof(double) * 3 * L);
    state_free(&S);
    return 0;
}

/* What build_system uses for every edge at one state: the residual, the robust weight inv_sigma_sq * rho'(chi2) and both Jacobians,
 * for the edges with level[e] == 0 (the others are left zero).  Test infrastructure: lets the tests check an independent restatement
 * of the three edge models edge by edge.  pose_cw / points: the state (NULL: the problem's own); level: NULL = every edge active;
 * robust: per-edge Huber switch (NULL: the problem's e_robust).  Returns the number of active edges. */
int orc_lba_linearize(const orc_lba_problem_t* P, const double* pose_cw, const double* points, const uint8_t* level, const uint8_t* robust,
                      double* err_out, double* weight_out, double* Ji_out, double* Jj_out) {
    orc_lba_problem_t Q = *P;
    if (pose_cw) Q.pose_cw = pose_cw;
    if (points) Q.points = points;
    lba_t S;
    state_init(&S, &Q);
    const int E = P->n_edges;
    int n = 0;
    for (int e = 0; e < E; ++e) {
        if (level) S.level[e] = level[e];
        if (robust) S.robust[e] = robust[e];
    }
    memset(err_out, 0, sizeof(double) * 3 * (size_t)E);
    memset(weight_out, 0, sizeof(double) * (size_t)E);
    memset(Ji_out, 0, sizeof(double) * 9 * (size_t)E);
    memset(Jj_out, 0, sizeof(double) * 18 * (size_t)E);
    compute_active_errors(&S);
    for (int e = 0; e < E; ++e) {
        if (S.level[e]) continue;
        ++n;
        edge_jacobians(&S, e, Ji_out + 9 * e, Jj_out + 18 * e);
        double rho1 = 1.0; /* as build_system */
        if (S.robust[e]) {
            const double e2 = edge_chi2(&S, e), delta = (double)P->e_delta[e];
            if (e2 > delta * delta) rho1 = delta / sqrt(e2);
        }
        weight_out[e] = (double)P->e_inv_sigma_sq[e] * rho1;
        memcpy(err_out + 3 * e, S.err + 3 * e, sizeof(double) * 3);
    }
    state_free(&S);
    return n;
}

/* optimize::global_bundle_adjuster (src/stella_vslam/optimize/global_bundle_adjuster.cc:26-192 optimize_impl, :258-420 optimize,
 * :201-256 optimize_for_initialization) on a flattened problem: the same vertices and reprojection edges as the local bundle adjuster
 * (every keyframe free except the spanning root, Huber on landmark edges when use_huber_kernel), ONE optimize(num_iter) with the
 * terminate action at `gain_threshold` (1e-3 in optimize(), the caller's value in optimize_for_initialization), no outlier pass.
 * g2o's LinearSolverCSparse there vs the dense Cholesky here: the same normal equations, the same solution up to rounding.
 * Returns 1 when aborted by the caller's flag (:340-342: set and not by the terminate action), else 0. */
int orc_global_ba_solve(const orc_lba_problem_t* P, int num_iter, double gain_threshold, volatile uint8_t* force_stop, double* pose_cw_out,
                        double* points_out, orc_lba_stats_t* stats) {
    lba_t S;
    state_init(&S, P);
    const int K = P->n_poses, L = P->n_points;
    if (stats) memset(stats, 0, sizeof(*stats));
    g_gain_thr = gain_threshold;
    const int n1 = optimize_rounds(&S, num_iter, force_stop, stats, 0);
    g_gain_thr = 1e-3;
    if (stats) stats->iterations[0] = n1;
    for (int k = 0; k < K; ++k) {
        double* M = pose_cw_out + 16 * k;
        if (P->pose_fixed[k]) {
            memcpy(M, P->pose_cw + 16 * k, sizeof(double) * 16);
            continue;
        }
        double R[9];
        quat_to_rot(S.q + 4 * k, R);
        M[0] = R[0]; M[1] = R[1]; M[2] = R[2]; M[3] = S.t[3 * k];
        M[4] = R[3]; M[5] = R[4]; M[6] = R[5]; M[7] = S.t[3 * k + 1];
        M[8] = R[6]; M[9] = R[7]; M[10] = R[8]; M[11] = S.t[3 * k + 2];
        M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
    }
    memcpy(points_out, S.pts, sizeof(double) * 3 * L);
    state_free(&S);
    return 0;
}

/* optimize::pose_optimizer_g2o::optimize (src/stella_vslam/optimize/pose_optimizer_g2o.cc:38-175) on a flattened frame: one free
 * pose, the landmarks it observes (fixed), one unary edge per observation (internal/se3/perspective_pose_opt_edge.h,
 * equirectangular_pose_opt_edge.h: the pose block of the corresponding reprojection edge), Huber(sqrt chi-square) on every edge.
 * P must hold n_poses = 1 (free), every point fixed, e_pose = 0.  Returns num_init_obs - num_bad_obs (0 if fewer than 5 edges). */
unsigned orc_pose_optimize(const orc_lba_problem_t* P, int num_trials_robust, int num_trials, int num_each_iter, double* pose_cw_out,
                           uint8_t* outlier_flags) {
    const int E = P->n_edges;
    memcpy(pose_cw_out, P->pose_cw, sizeof(double) * 16);
    for (int e = 0; e < E; ++e) outlier_flags[e] = 0;
    if (E < 5) return 0; /* :116-118 */
    lba_t S;
    state_init(&S, P);
    if (num_trials_robust == 0)
        for (int e = 0; e < E; ++e) S.robust[e] = 0; /* :123-127 */
    unsigned num_bad = 0;
    for (int trial = 0; trial < num_trials_robust + num_trials; ++trial) {
        optimize_rounds(&S, num_each_iter, NULL, NULL, 0); /* initializeOptimization (level-0 edges) + optimize(num_each_iter_) */
        num_bad = 0;
        for (int e = 0; e < E; ++e) {
            if (outlier_flags[e]) edge_error(&S, e, S.err + 3 * e, NULL); /* :137-139: inactive edges are re-evaluated at the new pose */
            const double thr = (edge_dim(P, e) == 2) ? (double)5.99146f : (double)7.81473f;
            if (thr < edge_chi2(&S, e)) {
                outlier_flags[e] = 1;
                S.level[e] = 1;
                ++num_bad;
            } else {
                outlier_flags[e] = 0;
                S.level[e] = 0;
            }
            if (num_trials != 0 && trial + 1 == num_trials_robust) S.robust[e] = 0; /* :164-166 */
        }
        if ((unsigned)E - num_bad < 5) break; /* :169-171 */
    }
    pose_to_mat(&S, 0, pose_cw_out);
    state_free(&S);
    return (unsigned)E - num_bad;
}
