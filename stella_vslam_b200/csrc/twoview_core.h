/* twoview_core.h -- the two-view RANSAC solvers of monocular initialisation: solve::homography_solver and solve::fundamental_solver
 * (src/stella_vslam/solve/homography_solver.cc, fundamental_solver.cc) with solve::normalize (solve/common.cc):
 *   normalize over all keypoints of a frame (float centroid and L1 deviation summed in order; cv::Point2f / double formed in double and
 *     rounded to float, as OpenCV's Point_ operator/= does; the 3 x 3 transform in double);
 *   compute_H_21: the 2n x 9 DLT, V's last column of its JacobiSVD, degenerate when rank() < 8;
 *   compute_F_21: the n x 9 eight-point matrix, V's last column, then the 3 x 3 JacobiSVD with sigma_3 = 0;
 *   check_inliers of both: H's symmetric transfer error (Eigen's 3 x 3 cofactor inverse, each squaredNorm rounded to float, the larger
 *     kept), F's Sampson distance in double; the float threshold chi_sq * sigma_sq and the float cost accumulated in match order with
 *     each branch's own mix of float and double;
 *   the denormalisation T2^-1 Hn T1 and T2^T Fn T1.
 * The n x 9 JacobiSVD (es_svd_n9), its rank() (es_svd_rank) and the rank-2 projection (es_rank2) are essential_core.h's, which the
 * includer includes first.
 *
 * One source, compiled twice: as device code by twoview_kernels.cu (explicit round-to-nearest intrinsics) and as C by
 * tests/twoview_oracle.c (-ffp-contract=off).  Besides essential_core.h's macros the includer defines
 *   tv_fa, tv_fs, tv_fm, tv_fd   correctly rounded float add, subtract, multiply, divide.
 * Points are float (x, y) pairs; matrices are row-major double. */

#define TV_MODEL_H 0
#define TV_MODEL_F 1

/* ---- solve::normalize ------------------------------------------------------------------------------------------------------- */

/* The sums of normalize over the n keypoints pts (n x 2): the float centroid mean, the float L1 deviation l1 and the transform T. */
ES_FN void tv_normalize_stats(int n, const float* pts, float* mean, float* l1, double* T) {
    float sx = 0.0f, sy = 0.0f;
    for (int i = 0; i < n; ++i) {  /* std::accumulate of cv::Point2f: float adds in order */
        sx = tv_fa(sx, pts[2 * i]);
        sy = tv_fa(sy, pts[2 * i + 1]);
    }
    mean[0] = (float)dd((double)sx, (double)n);  /* Point_<float> / double: formed in double, rounded to float */
    mean[1] = (float)dd((double)sy, (double)n);
    float lx = 0.0f, ly = 0.0f;
    for (int i = 0; i < n; ++i) {
        lx = tv_fa(lx, fabsf(tv_fs(pts[2 * i], mean[0])));
        ly = tv_fa(ly, fabsf(tv_fs(pts[2 * i + 1], mean[1])));
    }
    l1[0] = (float)dd((double)lx, (double)n);
    l1[1] = (float)dd((double)ly, (double)n);
    const double dx = (double)l1[0], dy = (double)l1[1];
    T[0] = dd(1.0, dx);
    T[1] = dd(0.0, dx);
    T[2] = dd((double)-mean[0], dx);
    T[3] = dd(0.0, dy);
    T[4] = dd(1.0, dy);
    T[5] = dd((double)-mean[1], dy);
    T[6] = 0.0;
    T[7] = 0.0;
    T[8] = 1.0;
}

/* One normalised point: (pt - mean) / l1 in float. */
ES_FN void tv_normalize_point(const float* pt, const float* mean, const float* l1, float* out) {
    out[0] = tv_fd(tv_fs(pt[0], mean[0]), l1[0]);
    out[1] = tv_fd(tv_fs(pt[1], mean[1]), l1[1]);
}

/* ---- 3 x 3 algebra ------------------------------------------------------------------------------------------------------------ */

/* Eigen's 3 x 3 inverse: cofactors of column 0, det = their dot with column 0, then every cofactor times 1 / det. */
ES_FN double tv_cof(const double* m, int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return ds(dm(m[i1 * 3 + j1], m[i2 * 3 + j2]), dm(m[i1 * 3 + j2], m[i2 * 3 + j1]));
}

ES_FN void tv_inverse33(const double* m, double* r) {
    const double c00 = tv_cof(m, 0, 0), c10 = tv_cof(m, 1, 0), c20 = tv_cof(m, 2, 0);
    const double det = da(da(dm(c00, m[0]), dm(c10, m[3])), dm(c20, m[6]));
    const double invdet = dd(1.0, det);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[i * 3 + j] = dm(tv_cof(m, j, i), invdet);
}

/* r = a b */
ES_FN void tv_mul33(const double* a, const double* b, double* r) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[i * 3 + j] = da(da(dm(a[i * 3], b[j]), dm(a[i * 3 + 1], b[3 + j])), dm(a[i * 3 + 2], b[6 + j]));
}

/* The left factor of the denormalisation: T2.inverse() for H, T2.transpose() for F. */
ES_FN void tv_left_factor(int model, const double* T2, double* D2) {
    if (model == TV_MODEL_H) {
        tv_inverse33(T2, D2);
    } else {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) D2[i * 3 + j] = T2[j * 3 + i];
    }
}

/* M = (D2 Mn) T1 */
ES_FN void tv_denormalise(const double* D2, const double* Mn, const double* T1, double* M) {
    double A[9];
    tv_mul33(D2, Mn, A);
    tv_mul33(A, T1, M);
}

/* ---- compute_H_21 / compute_F_21 ------------------------------------------------------------------------------------------------ */

/* The rows of one correspondence (normalised points p1, p2) in the coefficient matrix: two for H, one for F.  Returns the row count. */
ES_FN int tv_rows(int model, const float* p1, const float* p2, double* r) {
    const double x1 = (double)p1[0], y1 = (double)p1[1];
    if (model == TV_MODEL_H) {
        const double y2 = (double)p2[1], mx2 = (double)-p2[0];
        r[0] = 0.0, r[1] = 0.0, r[2] = 0.0;
        r[3] = -x1, r[4] = -y1, r[5] = -1.0;
        r[6] = dm(y2, x1), r[7] = dm(y2, y1), r[8] = dm(y2, 1.0);
        r[9] = x1, r[10] = y1, r[11] = 1.0;
        r[12] = 0.0, r[13] = 0.0, r[14] = 0.0;
        r[15] = dm(mx2, x1), r[16] = dm(mx2, y1), r[17] = dm(mx2, 1.0);
        return 2;
    }
    const double x2 = (double)p2[0], y2 = (double)p2[1];
    r[0] = dm(x2, x1), r[1] = dm(x2, y1), r[2] = dm(x2, 1.0);
    r[3] = dm(y2, x1), r[4] = dm(y2, y1), r[5] = dm(y2, 1.0);
    r[6] = x1, r[7] = y1, r[8] = 1.0;
    return 1;
}

/* compute_H_21 / compute_F_21 on the m correspondences sel[0..m-1] (match indices) of the normalised points n1, n2 (matches: n x 2
 * keypoint indices).  S is (2m or m) x 9 scratch.  Mn receives the normalised matrix.  Returns 1, or 0 when H's coefficient matrix has
 * rank() < 8 (Mn not written); *status gains ES_STATUS_SVD when a Jacobi SVD hit its sweep bound. */
ES_BIG int tv_estimate(int model, const float* n1, const float* n2, const int32_t* matches, const int32_t* sel, int m, double* S, double* Mn,
                       int* status) {
    const int per = model == TV_MODEL_H ? 2 : 1, rows = per * m;
    double scale = 0.0;
    for (int i = 0; i < m; ++i) {
        const int32_t q = sel[i];
        double* r = S + (size_t)i * 9 * per;
        tv_rows(model, n1 + 2 * (size_t)matches[2 * (size_t)q], n2 + 2 * (size_t)matches[2 * (size_t)q + 1], r);
        for (int k = 0; k < 9 * per; ++k) scale = es_max(scale, fabs(r[k]));
    }
    if (scale == 0.0) scale = 1.0;
    double v9[9];
    if (model == TV_MODEL_H) {
        double sv[9];
        int nonzero = 0;
        *status |= es_svd_n9(rows, S, scale, v9, sv, &nonzero);
        if (es_svd_rank(rows < 9 ? rows : 9, sv, nonzero) < 8) return 0;
        for (int k = 0; k < 9; ++k) Mn[k] = v9[k];
        return 1;
    }
    *status |= es_svd_n9(rows, S, scale, v9, NULL, NULL);
    *status |= es_rank2(v9, Mn);
    return 1;
}

/* ---- check_inliers ----------------------------------------------------------------------------------------------------------------- */

/* chi_sq * sigma_sq (chi_sq = 5.991f, sigma_sq = sigma * sigma), both float as the reference stores them */
ES_FN float tv_thr(float sigma) { return tv_fm(5.991f, tv_fm(sigma, sigma)); }

/* |p - H q / (H q)_z|^2 rounded to float (q, p homogeneous with z = 1) */
ES_FN float tv_transfer(const double* H, double qx, double qy, double px, double py) {
    double t[3];
    for (int r = 0; r < 3; ++r) t[r] = da(da(dm(H[r * 3], qx), dm(H[r * 3 + 1], qy)), dm(H[r * 3 + 2], 1.0));
    const double z = t[2];
    const double ex = ds(px, dd(t[0], z)), ey = ds(py, dd(t[1], z)), ez = ds(1.0, dd(t[2], z));
    return (float)da(da(dm(ex, ex), dm(ey, ey)), dm(ez, ez));
}

/* One match's term: *in = the inlier decision; returns what the branch adds to the cost (H: a float value either way; F: the double
 * Sampson distance for an inlier, the float threshold otherwise).  Mi is H_21.inverse() (unused for F). */
ES_FN double tv_term(int model, const double* M, const double* Mi, const float* k1, const float* k2, float thr, int* in) {
    const double x1 = (double)k1[0], y1 = (double)k1[1], x2 = (double)k2[0], y2 = (double)k2[1];
    if (model == TV_MODEL_H) {
        const float d1 = tv_transfer(M, x1, y1, x2, y2);
        const float d2 = tv_transfer(Mi, x2, y2, x1, y1);
        const float dist = (d1 < d2) ? d2 : d1;  /* std::max */
        *in = (double)thr > (double)dist;         /* double thr = chi_sq * sigma_sq; thr > dist_sq */
        return *in ? (double)dist : (double)thr;
    }
    double f1[3], f2[3];
    for (int r = 0; r < 3; ++r) f1[r] = da(da(dm(M[r * 3], x1), dm(M[r * 3 + 1], y1)), dm(M[r * 3 + 2], 1.0));
    for (int c = 0; c < 3; ++c) f2[c] = da(da(dm(x2, M[c]), dm(y2, M[3 + c])), dm(1.0, M[6 + c]));
    const double e = da(da(dm(f2[0], x1), dm(f2[1], y1)), dm(f2[2], 1.0));
    const double den = da(da(dm(f1[0], f1[0]), dm(f1[1], f1[1])), da(dm(f2[0], f2[0]), dm(f2[1], f2[1])));
    const double dist = dd(dm(e, e), den);
    *in = (double)thr > dist;
    return *in ? dist : (double)thr;
}

/* cost += term with the branch's types: H adds float to float either way; F adds the double distance to the float cost (formed in
 * double, rounded to float) or the float threshold in float. */
ES_FN float tv_accumulate(int model, float cost, double term, int in) {
    if (model == TV_MODEL_F && in) return (float)da((double)cost, term);
    return tv_fa(cost, (float)term);
}

/* check_inliers(M) over the n matches, in match order.  flags (may be null) receive the decisions. */
ES_FN unsigned tv_check_inliers(int model, const float* k1, const float* k2, const int32_t* matches, int n, const double* M, float sigma,
                                uint8_t* flags, float* cost) {
    double Mi[9];
    if (model == TV_MODEL_H) tv_inverse33(M, Mi);
    const float thr = tv_thr(sigma);
    unsigned num = 0;
    float c = 0.0f;
    for (int j = 0; j < n; ++j) {
        int in;
        const double t = tv_term(model, M, Mi, k1 + 2 * (size_t)matches[2 * (size_t)j], k2 + 2 * (size_t)matches[2 * (size_t)j + 1], thr, &in);
        c = tv_accumulate(model, c, t, in);
        num += (unsigned)in;
        if (flags) flags[j] = (uint8_t)in;
    }
    *cost = c;
    return num;
}
