/* initialize_core.h -- the reconstruction of monocular initialisation (src/stella_vslam/initialize/base.cc, perspective.cc,
 * bearing_vector.cc) with the decompositions it calls (solve/homography_solver.cc:142-249, fundamental_solver.cc:135-140,
 * essential_solver.cc:192-219) and the midpoint triangulation (solve/triangulator.h, the bearing overload):
 *   in_choose_H       perspective::initialize's rel_cost_H rule (NaN when both costs are 0: the F path runs);
 *   in_svd33          JacobiSVD<Mat33_t> with full U and V: scaled by the largest |entry|, no QR preconditioner (square), the sign of
 *                     negative singular values folded into U, descending sort (essential_core.h's svd_core sweeps);
 *   in_decompose_H    Faugeras' eight hypotheses from K2^-1 H K1, with the reference's float intermediates and its rank test;
 *   in_decompose_E    U's third column and U W V^T / U W^T V^T with their determinant sign fixed: {R1, R1, R2, R2}, {t, -t, t, -t};
 *   in_match          base::triangulate's body for one inlier match (midpoint, float parallax, depth tests, both reprojections);
 *   in_select         find_most_plausible_pose's rejection rules in the reference's order.
 * Products and sums run left to right in index order (Eigen's unrolled reductions are not reproduced).
 *
 * One source, compiled twice: as device code by initialize_kernels.cu and as C by tests/initialize_oracle.c (-ffp-contract=off).
 * Besides essential_core.h's and twoview_core.h's macros and functions (included first) the includer defines
 *   IN_FSQRT(x)                           correctly rounded float square root;
 *   in_cam_t                              one view's camera;
 *   int in_reproject(const in_cam_t* cam, const double* Rt, const double* p, double* q)
 *                                         camera::*::reproject_to_image of p under Rt (rotation row-major, then translation) into
 *                                         the pixel q; returns the visibility flag.
 * Matrices are row-major double. */

#define IN_MODEL_NONE 0
#define IN_MODEL_H 1
#define IN_MODEL_F 2
#define IN_MODEL_E 3

#define IN_STAGE_NO_MODEL 0
#define IN_STAGE_DECOMPOSE 1
#define IN_STAGE_MIN_VALID 2
#define IN_STAGE_AMBIGUOUS 3
#define IN_STAGE_PARALLAX 4
#define IN_STAGE_MIN_TRIANGULATED 5
#define IN_STAGE_SUCCEEDED 6

/* 0.5 > cost_H / (cost_H + cost_F) in float, and H valid */
ES_FN int in_choose_H(float cost_H, float cost_F, int valid_H) {
    const float rel = tv_fd(cost_H, tv_fa(cost_H, cost_F));
    return 0.5 > (double)rel && valid_H;
}

/* Eigen's 3 x 3 determinant: cofactor expansion along row 0 */
ES_FN double in_det33(const double* m) {
    return da(ds(dm(m[0], ds(dm(m[4], m[8]), dm(m[5], m[7]))), dm(m[1], ds(dm(m[3], m[8]), dm(m[5], m[6])))),
              dm(m[2], ds(dm(m[3], m[7]), dm(m[4], m[6]))));
}

ES_FN void in_transpose33(const double* a, double* r) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[i * 3 + j] = a[j * 3 + i];
}

/* r = a v */
ES_FN void in_mul33v(const double* a, const double* v, double* r) {
    for (int i = 0; i < 3; ++i) r[i] = da(da(dm(a[i * 3], v[0]), dm(a[i * 3 + 1], v[1])), dm(a[i * 3 + 2], v[2]));
}

ES_FN double in_dot3(const double* a, const double* b) { return da(da(dm(a[0], b[0]), dm(a[1], b[1])), dm(a[2], b[2])); }

/* JacobiSVD<Mat33_t>(A, ComputeFullU | ComputeFullV): A = U diag(s) V^T.  Returns 0, or ES_STATUS_SVD when the sweeps hit their bound. */
ES_BIG int in_svd33(const double* A, double* U, double* s, double* V) {
    double W[9];
    double sc = 0.0;
    for (int k = 0; k < 9; ++k) sc = es_max(sc, fabs(A[k]));
    if (sc == 0.0) sc = 1.0;
    for (int k = 0; k < 9; ++k) {
        W[k] = dd(A[k], sc);
        U[k] = V[k] = (k % 4 == 0) ? 1.0 : 0.0;
    }
    return svd_core(3, W, 3, U, V, sc, s) < 0 ? ES_STATUS_SVD : 0;
}

/* One hypothesis of the H decomposition: R = (s U) aux_rot V^T, t = U aux_trans / |U aux_trans|, n = +-V aux_normal (n_z >= 0). */
ES_FN void in_h_pose(const double* sU, const double* U, const double* V, const double* Vt, const double* aux_rot, double tx, double tz, double tf,
                     double nx, double nz, double* R, double* t, double* nrm) {
    double T[9];
    tv_mul33(sU, aux_rot, T);
    tv_mul33(T, Vt, R);
    const double at[3] = {dm(tx, tf), dm(0.0, tf), dm(tz, tf)};
    double u[3];
    in_mul33v(U, at, u);
    const double norm = ES_SQRT(in_dot3(u, u));
    for (int k = 0; k < 3; ++k) t[k] = dd(u[k], norm);
    const double an[3] = {nx, 0.0, nz};
    in_mul33v(V, an, nrm);
    if (nrm[2] < 0.0)
        for (int k = 0; k < 3; ++k) nrm[k] = -nrm[k];
}

/* homography_solver::decompose(H_21, K1, K2): 8 rotations (R: 8 x 9), unit translations (t: 8 x 3) and plane normals (nrm: 8 x 3).
 * Returns 0 when the rank test rejects (nothing written).  *status gains ES_STATUS_SVD. */
ES_BIG int in_decompose_H(const double* H, const double* K1, const double* K2, double* R, double* t, double* nrm, int* status) {
    double K2i[9], T[9], A[9], U[9], V[9], Vt[9], lam[3];
    tv_inverse33(K2, K2i);
    tv_mul33(K2i, H, T);
    tv_mul33(T, K1, A);
    *status |= in_svd33(A, U, lam, V);
    in_transpose33(V, Vt);
    const float d1 = (float)lam[0], d2 = (float)lam[1], d3 = (float)lam[2];
    if ((double)tv_fd(d1, d2) < 1.0001 || (double)tv_fd(d2, d3) < 1.0001) return 0;
    const float s = (float)dm(in_det33(U), in_det33(Vt));
    const float d1s = tv_fm(d1, d1), d2s = tv_fm(d2, d2), d3s = tv_fm(d3, d3);
    const float aux_1 = IN_FSQRT(tv_fd(tv_fs(d1s, d2s), tv_fs(d1s, d3s)));
    const float aux_3 = IN_FSQRT(tv_fd(tv_fs(d2s, d3s), tv_fs(d1s, d3s)));
    const float x1s[4] = {aux_1, aux_1, -aux_1, -aux_1};
    const float x3s[4] = {aux_3, -aux_3, aux_3, -aux_3};
    const float root = IN_FSQRT(tv_fm(tv_fs(d1s, d2s), tv_fs(d2s, d3s)));
    double sU[9];
    for (int k = 0; k < 9; ++k) sU[k] = dm((double)s, U[k]);
    /* d' > 0: Eq. (13), (14) */
    const float den_p = tv_fm(tv_fa(d1, d3), d2);
    const float sin_theta = tv_fd(root, den_p);
    const float cos_theta = tv_fd(tv_fa(d2s, tv_fm(d1, d3)), den_p);
    const float sin_thetas[4] = {sin_theta, -sin_theta, -sin_theta, sin_theta};
    const float d13m = tv_fs(d1, d3), d13p = tv_fa(d1, d3);
    for (int i = 0; i < 4; ++i) {
        const double aux[9] = {(double)cos_theta, 0.0, (double)-sin_thetas[i], 0.0, 1.0, 0.0, (double)sin_thetas[i], 0.0, (double)cos_theta};
        in_h_pose(sU, U, V, Vt, aux, (double)x1s[i], -(double)x3s[i], (double)d13m, (double)x1s[i], (double)x3s[i], R + 9 * i, t + 3 * i,
                  nrm + 3 * i);
    }
    /* d' < 0: Eq. (15), (16) */
    const float den_m = tv_fm(tv_fs(d1, d3), d2);
    const float sin_phi = tv_fd(root, den_m);
    const float cos_phi = tv_fd(tv_fs(tv_fm(d1, d3), d2s), den_m);
    const float sin_phis[4] = {sin_phi, -sin_phi, -sin_phi, sin_phi};
    for (int i = 0; i < 4; ++i) {
        const double aux[9] = {(double)cos_phi, 0.0, (double)sin_phis[i], 0.0, -1.0, 0.0, (double)sin_phis[i], 0.0, (double)-cos_phi};
        in_h_pose(sU, U, V, Vt, aux, (double)x1s[i], (double)x3s[i], (double)d13p, (double)x1s[i], (double)x3s[i], R + 9 * (4 + i),
                  t + 3 * (4 + i), nrm + 3 * (4 + i));
    }
    return 1;
}

/* fundamental_solver::decompose's E_21 = K2^T F_21 K1 */
ES_FN void in_essential_of_F(const double* F, const double* K1, const double* K2, double* E) {
    double K2t[9], T[9];
    in_transpose33(K2, K2t);
    tv_mul33(K2t, F, T);
    tv_mul33(T, K1, E);
}

/* essential_solver::decompose(E_21): R (4 x 9) = {R1, R1, R2, R2}, t (4 x 3) = {t, -t, t, -t}.  *status gains ES_STATUS_SVD. */
ES_BIG void in_decompose_E(const double* E, double* R, double* t, int* status) {
    double U[9], V[9], Vt[9], s[3], T[9], R1[9], R2[9];
    const double W[9] = {0.0, -1.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0};
    const double Wt[9] = {0.0, 1.0, 0.0, -1.0, 0.0, 0.0, 0.0, 0.0, 1.0};
    *status |= in_svd33(E, U, s, V);
    in_transpose33(V, Vt);
    double tr[3] = {U[2], U[5], U[8]};
    const double z = in_dot3(tr, tr);
    if (z > 0.0) {
        const double nz = ES_SQRT(z);
        for (int k = 0; k < 3; ++k) tr[k] = dd(tr[k], nz);
    }
    tv_mul33(U, W, T);
    tv_mul33(T, Vt, R1);
    if (in_det33(R1) < 0.0)
        for (int k = 0; k < 9; ++k) R1[k] = dm(R1[k], -1.0);
    tv_mul33(U, Wt, T);
    tv_mul33(T, Vt, R2);
    if (in_det33(R2) < 0.0)
        for (int k = 0; k < 9; ++k) R2[k] = dm(R2[k], -1.0);
    for (int h = 0; h < 4; ++h) {
        for (int k = 0; k < 9; ++k) R[9 * h + k] = h < 2 ? R1[k] : R2[k];
        for (int k = 0; k < 3; ++k) t[3 * h + k] = (h & 1) ? -tr[k] : tr[k];
    }
}

/* -R^T t: trans_12 of the triangulator, and the current camera's centre in base::triangulate */
ES_FN void in_neg_rt_t(const double* R, const double* t, double* c) {
    for (int i = 0; i < 3; ++i) c[i] = -da(da(dm(R[i], t[0]), dm(R[3 + i], t[1])), dm(R[6 + i], t[2]));
}

/* triangulator::triangulate(bearing_1, bearing_2, rot_21, trans_21): the midpoint of the closest points of the two rays, in frame 1 */
ES_FN void in_midpoint(const double* b1, const double* b2, const double* R, const double* t, double* p) {
    double t12[3], b21[3];
    in_neg_rt_t(R, t, t12);
    for (int i = 0; i < 3; ++i) b21[i] = da(da(dm(R[i], b2[0]), dm(R[3 + i], b2[1])), dm(R[6 + i], b2[2]));
    const double a00 = in_dot3(b1, b1), a10 = in_dot3(b1, b21), a01 = -a10, a11 = -in_dot3(b21, b21);
    const double c0 = in_dot3(b1, t12), c1 = in_dot3(b21, t12);
    const double invdet = dd(1.0, ds(dm(a00, a11), dm(a10, a01)));  /* Eigen's 2 x 2 inverse */
    const double i00 = dm(a11, invdet), i10 = dm(-a10, invdet), i01 = dm(-a01, invdet), i11 = dm(a00, invdet);
    const double l0 = da(dm(i00, c0), dm(i01, c1)), l1 = da(dm(i10, c0), dm(i11, c1));
    for (int k = 0; k < 3; ++k) p[k] = dd(da(dm(l0, b1[k]), da(dm(l1, b21[k]), t12[k])), 2.0);
}

/* |q - k|^2 rounded to float (Vec2_t - cv::Point2f, squaredNorm) */
ES_FN float in_err_sq(const double* q, const float* k) {
    const double e0 = ds(q[0], (double)k[0]), e1 = ds(q[1], (double)k[1]);
    return (float)da(dm(e0, e0), dm(e1, e1));
}

#define IN_TRI_REJECTED 0
#define IN_TRI_VALID 1         /* valid, parallax too small to count as triangulated */
#define IN_TRI_TRIANGULATED 2

/* base::triangulate's body (base.cc:138-199) for one inlier match with bearings b1 / b2 and undistorted keypoints k1 / k2 under the
 * hypothesis Rt (rotation row-major, then translation); ctr is -R^T t.  Returns IN_TRI_*; p receives the point, *cos_parallax its
 * float parallax cosine (both meaningful unless rejected).  The reference reads an unset pixel when a small-parallax point lies behind
 * a perspective camera; the projection computed by in_reproject is used there. */
ES_FN int in_match(const in_cam_t* cam_ref, const in_cam_t* cam_cur, const double* Rt, const double* ctr, int depth_is_positive, float thr_sq,
                   const double* b1, const double* b2, const float* k1, const float* k2, double* p, float* cos_parallax) {
    in_midpoint(b1, b2, Rt, Rt + 9, p);
    if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2])) return IN_TRI_REJECTED;
    const double cn[3] = {ds(p[0], ctr[0]), ds(p[1], ctr[1]), ds(p[2], ctr[2])};
    const float ref_norm = (float)ES_SQRT(in_dot3(p, p));
    const float cur_norm = (float)ES_SQRT(in_dot3(cn, cn));
    const float cp = (float)dd(in_dot3(p, cn), (double)tv_fm(ref_norm, cur_norm));
    const int small = (float)0.99996192306 < cp;  /* cos(0.5 deg) */
    if (depth_is_positive && !small) {
        if (p[2] <= 0.0) return IN_TRI_REJECTED;
        if (da(da(da(dm(Rt[6], p[0]), dm(Rt[7], p[1])), dm(Rt[8], p[2])), Rt[11]) <= 0.0) return IN_TRI_REJECTED;
    }
    const double ident[12] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};
    double q[2];
    if (!in_reproject(cam_ref, ident, p, q) && !small) return IN_TRI_REJECTED;
    if (thr_sq < in_err_sq(q, k1)) return IN_TRI_REJECTED;
    if (!in_reproject(cam_cur, Rt, p, q) && !small) return IN_TRI_REJECTED;
    if (thr_sq < in_err_sq(q, k2)) return IN_TRI_REJECTED;
    *cos_parallax = cp;
    return small ? IN_TRI_VALID : IN_TRI_TRIANGULATED;
}

/* find_most_plausible_pose's rules (base.cc:63-87) over n_hyp hypotheses; cos_thr = cos(parallax_deg_thr / 180 pi) in double.
 * Returns IN_STAGE_MIN_VALID .. IN_STAGE_SUCCEEDED; *best the first hypothesis with the most valid points. */
ES_FN int in_select(int n_hyp, const int32_t* nums_valid, const int32_t* num_triangulated, const float* parallax_cos, uint32_t min_num_valid_pts,
                    uint32_t min_num_triangulated, double cos_thr, int* best) {
    int b = 0;
    for (int i = 1; i < n_hyp; ++i)
        if (nums_valid[i] > nums_valid[b]) b = i;
    *best = b;
    if ((uint32_t)nums_valid[b] < min_num_valid_pts) return IN_STAGE_MIN_VALID;
    int similar = 0;
    for (int i = 0; i < n_hyp; ++i)
        if (dm(0.8, (double)nums_valid[b]) < (double)nums_valid[i]) ++similar;
    if (1 < similar) return IN_STAGE_AMBIGUOUS;
    if ((double)parallax_cos[b] > cos_thr) return IN_STAGE_PARALLAX;
    if ((uint32_t)num_triangulated[b] < min_num_triangulated) return IN_STAGE_MIN_TRIANGULATED;
    return IN_STAGE_SUCCEEDED;
}
