/*
 * tests/mapping_oracle.c -- TEST INFRASTRUCTURE.  CPU restatement of the two-view triangulation of the mapping module:
 *   module::two_view_triangulator          src/stella_vslam/module/two_view_triangulator.{h,cc}
 *   solve::triangulator::triangulate       src/stella_vslam/solve/triangulator.h:77-90 (4x4 Eigen::JacobiSVD, column 3 of V)
 *   data::triangulate_stereo               src/stella_vslam/data/common.cc:192-260
 *   camera::{perspective,equirectangular}::reproject_to_image
 * It defines the evaluation order the device code follows: sums left to right in index order, no contraction (built with
 * -ffp-contract=off), float where the reference stores float.  The Jacobi SVD follows Eigen's JacobiSVD for a square fixed-size
 * matrix: scale by the largest |a_ij|, no QR preconditioner, sweeps of real 2x2 SVDs (real_2x2_jacobi_svd + makeJacobi) until every
 * off-diagonal pair is <= max(DBL_MIN, 2 eps max|diag|), then |diag| sorted descending with the columns of V.
 */
#define _GNU_SOURCE
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

#define ORC_TRI_MAX_SWEEPS 64

/* Same layout as b200_tri_keyframe_t (include/b200vslam.h). */
typedef struct {
    double pose_cw[16], pose_wc[16]; /* row-major 4x4 */
    int32_t model;                   /* 0 perspective family, 1 equirectangular */
    double fx, fy, cx, cy, fx_inv, fy_inv, focal_x_baseline, true_baseline, cols, rows;
    float scale_factor;
    int32_t num_levels;
    const float* scale_factors;
    const float* level_sigma_sq;
    int32_t n_keypoints;
    const float* x;
    const float* y;
    const int32_t* octave;
    const float* x_right; /* NULL = monocular */
    const float* depth;   /* NULL = none */
    const double* bearings;
} orc_tri_keyframe_t;

/* apply_rotation_in_the_plane(x, y, (c, s)) on two 4-vectors with strides */
static void rot_plane(double* x, double* y, int stride, double c, double s) {
    if (c == 1.0 && s == 0.0) return;
    for (int i = 0; i < 4; ++i) {
        const double xi = x[i * stride], yi = y[i * stride];
        x[i * stride] = c * xi + s * yi;
        y[i * stride] = -s * xi + c * yi;
    }
}

/* Null vector (V column of the smallest singular value) of a row-major 4x4 matrix.  Returns the sweep count, or -1 when the
 * sweeps did not converge within ORC_TRI_MAX_SWEEPS. */
int orc_jacobi_svd4_null(const double* A_in, double* v_out) {
    double W[16], V[16], sv[4];
    double scale = 0.0;
    for (int k = 0; k < 16; ++k)
        if (fabs(A_in[k]) > scale) scale = fabs(A_in[k]);
    if (scale == 0.0) scale = 1.0;
    for (int k = 0; k < 16; ++k) {
        W[k] = A_in[k] / scale;
        V[k] = (k % 5 == 0) ? 1.0 : 0.0;
    }
    double max_diag = fabs(W[0]);
    for (int i = 1; i < 4; ++i)
        if (fabs(W[i * 5]) > max_diag) max_diag = fabs(W[i * 5]);
    const double precision = 2.0 * DBL_EPSILON;
    int sweeps = 0, finished = 0;
    while (!finished) {
        if (sweeps == ORC_TRI_MAX_SWEEPS) return -1;
        ++sweeps;
        finished = 1;
        for (int p = 1; p < 4; ++p) {
            for (int q = 0; q < p; ++q) {
                const double pm = precision * max_diag;
                const double threshold = DBL_MIN < pm ? pm : DBL_MIN;
                if (!(fabs(W[p * 4 + q]) > threshold || fabs(W[q * 4 + p]) > threshold)) continue;
                finished = 0;
                /* real_2x2_jacobi_svd */
                double m00 = W[p * 4 + p], m01 = W[p * 4 + q], m10 = W[q * 4 + p], m11 = W[q * 4 + q];
                double c1 = 1.0, s1 = 0.0;
                const double t = m00 + m11, d = m10 - m01;
                if (!(fabs(d) < DBL_MIN)) {
                    const double u = t / d;
                    const double tmp = sqrt(1.0 + u * u);
                    s1 = 1.0 / tmp;
                    c1 = u / tmp;
                }
                if (!(c1 == 1.0 && s1 == 0.0)) { /* m.applyOnTheLeft(0, 1, rot1) */
                    const double a0 = m00, a1 = m01, b0 = m10, b1 = m11;
                    m00 = c1 * a0 + s1 * b0;
                    m10 = -s1 * a0 + c1 * b0;
                    m01 = c1 * a1 + s1 * b1;
                    m11 = -s1 * a1 + c1 * b1;
                }
                /* j_right.makeJacobi(m00, m01, m11) */
                double cr = 1.0, sr = 0.0;
                const double deno = 2.0 * fabs(m01);
                if (!(deno < DBL_MIN)) {
                    const double tau = (m00 - m11) / deno;
                    const double w = sqrt(tau * tau + 1.0);
                    const double tt = tau > 0.0 ? 1.0 / (tau + w) : 1.0 / (tau - w);
                    const double sign_t = tt > 0.0 ? 1.0 : -1.0;
                    const double n = 1.0 / sqrt(tt * tt + 1.0);
                    sr = -sign_t * (m01 / fabs(m01)) * fabs(tt) * n;
                    cr = n;
                }
                /* j_left = rot1 * j_right^T, j_right^T = (cr, -sr) */
                const double cl = c1 * cr - s1 * -sr;
                const double sl = c1 * -sr + s1 * cr;
                rot_plane(W + p * 4, W + q * 4, 1, cl, sl);    /* applyOnTheLeft(p, q, j_left): rows */
                rot_plane(W + p, W + q, 4, cr, -sr);           /* applyOnTheRight(p, q, j_right): columns, with j_right^T */
                rot_plane(V + p, V + q, 4, cr, -sr);
                const double dp = fabs(W[p * 5]), dq = fabs(W[q * 5]);
                const double dm = dp < dq ? dq : dp;
                if (max_diag < dm) max_diag = dm;
            }
        }
    }
    for (int i = 0; i < 4; ++i) sv[i] = fabs(W[i * 5]) * scale;
    for (int i = 0; i < 4; ++i) {
        int pos = i;
        for (int k = i + 1; k < 4; ++k)
            if (sv[k] > sv[pos]) pos = k;
        if (sv[pos] == 0.0) break;
        if (pos != i) {
            const double ts = sv[i];
            sv[i] = sv[pos];
            sv[pos] = ts;
            for (int r = 0; r < 4; ++r) {
                const double tv = V[r * 4 + i];
                V[r * 4 + i] = V[r * 4 + pos];
                V[r * 4 + pos] = tv;
            }
        }
    }
    for (int r = 0; r < 4; ++r) v_out[r] = V[r * 4 + 3];
    return sweeps;
}

static double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

/* pose: row-major 4x4; R p + t, row by row */
static void transform(const double* pose, const double* p, double* out) {
    for (int r = 0; r < 3; ++r) out[r] = pose[r * 4] * p[0] + pose[r * 4 + 1] * p[1] + pose[r * 4 + 2] * p[2] + pose[r * 4 + 3];
}

/* rot_wc * b with rot_wc = rot_cw^T */
static void rotate_to_world(const double* pose_cw, const double* b, double* out) {
    for (int i = 0; i < 3; ++i) out[i] = pose_cw[i] * b[0] + pose_cw[4 + i] * b[1] + pose_cw[8 + i] * b[2];
}

static int depth_is_positive(const orc_tri_keyframe_t* K, const double* p) {
    const double* P = K->pose_cw;
    const double z = P[8] * p[0] + P[9] * p[1] + P[10] * p[2] + P[11];
    return K->model == 1 || 0.0 < z;
}

static int reprojection_ok(const orc_tri_keyframe_t* K, const double* p, int idx, int is_stereo) {
    double pc[3], r0, r1;
    float x_right_c;
    transform(K->pose_cw, p, pc);
    if (K->model == 1) {
        const double n = pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2];
        double b[3] = {pc[0], pc[1], pc[2]};
        if (n > 0.0) {
            const double s = sqrt(n);
            for (int k = 0; k < 3; ++k) b[k] = pc[k] / s;
        }
        const double latitude = -asin(b[1]);
        const double longitude = atan2(b[0], b[2]);
        r0 = K->cols * (0.5 + longitude / (2.0 * M_PI));
        r1 = K->rows * (0.5 - latitude / M_PI);
        x_right_c = 0.0f;
    } else {
        const double z_inv = 1.0 / pc[2];
        r0 = K->fx * pc[0] * z_inv + K->cx;
        r1 = K->fy * pc[1] * z_inv + K->cy;
        x_right_c = (float)(r0 - K->focal_x_baseline * z_inv);
    }
    const float sigma_sq = K->level_sigma_sq[K->octave[idx]];
    const double e0 = r0 - (double)K->x[idx], e1 = r1 - (double)K->y[idx];
    if (is_stereo) {
        const float exr = x_right_c - K->x_right[idx];
        const float chi = 7.81473f * sigma_sq;
        return !((double)chi < (e0 * e0 + e1 * e1) + (double)(exr * exr));
    }
    const float chi = 5.99146f * sigma_sq;
    return !((double)chi < e0 * e0 + e1 * e1);
}

static void triangulate_stereo(const orc_tri_keyframe_t* K, int idx, double* p) {
    const float depth = K->depth ? K->depth[idx] : -1.0f;
    if (!(0.0 < depth)) {
        p[0] = p[1] = p[2] = 0.0;
        return;
    }
    const float ux = (float)(((double)K->x[idx] - K->cx) * (double)depth * K->fx_inv);
    const float uy = (float)(((double)K->y[idx] - K->cy) * (double)depth * K->fy_inv);
    const double pc[3] = {ux, uy, depth};
    transform(K->pose_wc, pc, p);
}

/* two_view_triangulator::triangulate for one match.  pos_w gets the triangulated point (zeros when no branch applies) whatever
 * the outcome.  Returns 1 = accepted, 0 = rejected, -1 = the Jacobi sweeps did not converge. */
int orc_two_view_triangulate(const orc_tri_keyframe_t* k1, const orc_tri_keyframe_t* k2, int i1, int i2, float cos_rays_parallax_thr,
                             float ratio_factor, double* pos_w) {
    const float xr1 = k1->x_right ? k1->x_right[i1] : -1.0f, xr2 = k2->x_right ? k2->x_right[i2] : -1.0f;
    const int st1 = 0 <= xr1, st2 = 0 <= xr2;
    const double* b1 = k1->bearings + (size_t)i1 * 3;
    const double* b2 = k2->bearings + (size_t)i2 * 3;
    double rw1[3], rw2[3];
    rotate_to_world(k1->pose_cw, b1, rw1);
    rotate_to_world(k2->pose_cw, b2, rw2);
    const double cos_rays = dot3(rw1, rw2);
    const float d1 = k1->depth ? k1->depth[i1] : -1.0f, d2 = k2->depth ? k2->depth[i2] : -1.0f;
    const double cs1 = st1 ? cos(2.0 * atan2(k1->true_baseline / 2.0, (double)d1)) : 2.0;
    const double cs2 = st2 ? cos(2.0 * atan2(k2->true_baseline / 2.0, (double)d2)) : 2.0;
    const double cs = cs2 < cs1 ? cs2 : cs1;
    pos_w[0] = pos_w[1] = pos_w[2] = 0.0;
    const int two_cameras = ((!st1 && !st2) && 0.0 < cos_rays && cos_rays < (double)cos_rays_parallax_thr)
                            || ((st1 || st2) && 0.0 < cos_rays && cos_rays < cs);
    if (two_cameras) {
        const double *P1 = k1->pose_cw, *P2 = k2->pose_cw;
        double A[16], v[4];
        for (int j = 0; j < 4; ++j) {
            A[j] = b1[0] * P1[8 + j] - b1[2] * P1[j];
            A[4 + j] = b1[1] * P1[8 + j] - b1[2] * P1[4 + j];
            A[8 + j] = b2[0] * P2[8 + j] - b2[2] * P2[j];
            A[12 + j] = b2[1] * P2[8 + j] - b2[2] * P2[4 + j];
        }
        if (orc_jacobi_svd4_null(A, v) < 0) return -1;
        for (int k = 0; k < 3; ++k) pos_w[k] = v[k] / v[3];
    } else if (st1 && cs1 < cs2) {
        triangulate_stereo(k1, i1, pos_w);
    } else if (st2 && cs2 < cs1) {
        triangulate_stereo(k2, i2, pos_w);
    } else {
        return 0;
    }
    if (!depth_is_positive(k1, pos_w) || !depth_is_positive(k2, pos_w)) return 0;
    if (!reprojection_ok(k1, pos_w, i1, st1) || !reprojection_ok(k2, pos_w, i2, st2)) return 0;
    const double c1[3] = {k1->pose_wc[3], k1->pose_wc[7], k1->pose_wc[11]};
    const double c2[3] = {k2->pose_wc[3], k2->pose_wc[7], k2->pose_wc[11]};
    const double v1[3] = {pos_w[0] - c1[0], pos_w[1] - c1[1], pos_w[2] - c1[2]};
    const double v2[3] = {pos_w[0] - c2[0], pos_w[1] - c2[1], pos_w[2] - c2[2]};
    const double dist1 = sqrt(dot3(v1, v1)), dist2 = sqrt(dot3(v2, v2));
    if (dist1 == 0.0 || dist2 == 0.0) return 0;
    const double ratio_dists = dist2 / dist1;
    const float ratio_octave = k1->scale_factors[k1->octave[i1]] / k2->scale_factors[k2->octave[i2]];
    return (double)ratio_octave / ratio_dists < (double)ratio_factor && ratio_dists / (double)ratio_octave < (double)ratio_factor;
}

/* The constructor's constants (two_view_triangulator.cc:15-16). */
void orc_triangulator_constants(const orc_tri_keyframe_t* k1, const orc_tri_keyframe_t* k2, float rays_parallax_deg_thr, float* cos_thr,
                                float* ratio_factor) {
    *ratio_factor = 2.0f * (k1->scale_factor < k2->scale_factor ? k2->scale_factor : k1->scale_factor);
    *cos_thr = (float)cos(rays_parallax_deg_thr * M_PI / 180.0);
}

/* Every match of one keyframe pair.  matches: n x (idx_1, idx_2).  Returns the number accepted, -1 on a bad index / octave / an
 * equirectangular stereo keypoint (nothing written), -2 when an SVD did not converge. */
int orc_triangulate_pairs(const orc_tri_keyframe_t* k1, const orc_tri_keyframe_t* k2, float rays_parallax_deg_thr, int n,
                          const int32_t* matches, double* pos_w, uint8_t* ok) {
    for (int m = 0; m < n; ++m) {
        const int i1 = matches[2 * m], i2 = matches[2 * m + 1];
        if (i1 < 0 || i1 >= k1->n_keypoints || i2 < 0 || i2 >= k2->n_keypoints) return -1;
        if (k1->octave[i1] < 0 || k1->octave[i1] >= k1->num_levels || k2->octave[i2] < 0 || k2->octave[i2] >= k2->num_levels) return -1;
        if ((k1->model == 1 && k1->x_right && k1->x_right[i1] >= 0.0f) || (k2->model == 1 && k2->x_right && k2->x_right[i2] >= 0.0f)) return -1;
    }
    float cos_thr, ratio_factor;
    orc_triangulator_constants(k1, k2, rays_parallax_deg_thr, &cos_thr, &ratio_factor);
    int n_ok = 0;
    for (int m = 0; m < n; ++m) {
        const int r = orc_two_view_triangulate(k1, k2, matches[2 * m], matches[2 * m + 1], cos_thr, ratio_factor, pos_w + 3 * (size_t)m);
        if (r < 0) return -2;
        ok[m] = (uint8_t)r;
        n_ok += r;
    }
    return n_ok;
}
