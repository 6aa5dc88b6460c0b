/* twoview_oracle.c -- CPU restatement of solve::homography_solver::find_via_ransac and solve::fundamental_solver::find_via_ransac
 * (src/stella_vslam/solve/homography_solver.cc, fundamental_solver.cc).  The arithmetic is stella_vslam_b200/csrc/twoview_core.h
 * (on essential_core.h and the SVD / Householder pieces of tests/pnp_oracle.c, included, not copied) compiled as C here
 * (-ffp-contract=off); the RANSAC loop below follows the reference's control flow directly.  The entry points also expose the stages
 * (normalisation, coefficient matrices and their null vectors, the per-match errors) so the tests can check them against numpy.
 * Test infrastructure, compiled on first use. */
#include "pnp_oracle.c"

#include <stdlib.h>

#define ES_FN static
#define ES_BIG static
#define ES_SQRT(x) sqrt(x)
#define ES_MAKE_HOUSEHOLDER(v, len, stride, tau, beta) make_householder((v), (len), (stride), &(tau), &(beta))
static inline float tv_fa(float a, float b) { return a + b; }
static inline float tv_fs(float a, float b) { return a - b; }
static inline float tv_fm(float a, float b) { return a * b; }
static inline float tv_fd(float a, float b) { return a / b; }
#include "../stella_vslam_b200/csrc/essential_core.h"
#include "../stella_vslam_b200/csrc/twoview_core.h"

/* solve::normalize over n keypoints: normalised points (n x 2), mean, l1 and the transform */
void orc_normalize(int n, const float* pts, float* out, float* mean, float* l1, double* T) {
    tv_normalize_stats(n, pts, mean, l1, T);
    for (int i = 0; i < n; ++i) tv_normalize_point(pts + 2 * (size_t)i, mean, l1, out + 2 * (size_t)i);
}

/* compute_H_21 / compute_F_21 over m correspondences of (already normalised) points p1, p2 (m x 2).  Returns 1, 0 when H is
 * degenerate; *status the ES_STATUS_SVD bit. */
int orc_estimate(int model, int m, const float* p1, const float* p2, double* Mn, int* status) {
    int32_t* matches = (int32_t*)malloc(sizeof(int32_t) * 2 * (size_t)(m > 0 ? m : 1));
    int32_t* sel = (int32_t*)malloc(sizeof(int32_t) * (size_t)(m > 0 ? m : 1));
    double* S = (double*)malloc(sizeof(double) * 18 * (size_t)(m > 0 ? m : 1));
    for (int i = 0; i < m; ++i) matches[2 * i] = matches[2 * i + 1] = sel[i] = i;
    *status = 0;
    const int ok = tv_estimate(model, p1, p2, matches, sel, m, S, Mn, status);
    free(matches);
    free(sel);
    free(S);
    return ok;
}

/* JacobiSVD<Matrix<double, Dynamic, 9>> of the m x 9 A: V's last column, the singular values and rank().  Returns the status bits. */
int orc_svd_n9(int m, const double* A, double* v9, double* sv, int* rank) {
    double* S = (double*)malloc(sizeof(double) * 9 * (size_t)m);
    double scale = 0.0;
    for (int k = 0; k < 9 * m; ++k) {
        S[k] = A[k];
        scale = es_max(scale, fabs(A[k]));
    }
    if (scale == 0.0) scale = 1.0;
    int nonzero = 0;
    const int st = es_svd_n9(m, S, scale, v9, sv, &nonzero);
    *rank = es_svd_rank(m < 9 ? m : 9, sv, nonzero);
    free(S);
    return st;
}

void orc_inverse33(const double* m, double* r) { tv_inverse33(m, r); }

/* check_inliers(M) over n matches: count, flags and the float cost */
unsigned orc_check_inliers(int model, const float* k1, const float* k2, int n, const int32_t* matches, const double* M, float sigma,
                           uint8_t* flags, float* cost) {
    return tv_check_inliers(model, k1, k2, matches, n, M, sigma, flags, cost);
}

/* one match's error: H's symmetric transfer error (float) or F's Sampson distance (double), before thresholding */
double orc_error(int model, const double* M, const float* k1, const float* k2) {
    double Mi[9];
    if (model == TV_MODEL_H) tv_inverse33(M, Mi);
    int in;
    /* a threshold no finite error reaches makes every match an inlier, so the term is the error itself */
    return tv_term(model, M, Mi, k1, k2, FLT_MAX, &in);
}

/* find_via_ransac(max_num_iter = n_iter, recompute) on the given minimal sets (n_iter x 4 for H, x 8 for F).  Outputs as
 * b200_twoview_problem_t; flags untouched on the early return.  Returns the status bits. */
int orc_twoview_ransac(int model, int n1, const float* kp1, int n2, const float* kp2, int n, const int32_t* matches, float sigma, int n_iter,
                       int recompute, const int32_t* min_sets, int* valid, int* best_iter, int* num_inliers, float* best_cost, double* M_21,
                       uint8_t* flags) {
    const int set_size = model == TV_MODEL_H ? 4 : 8;
    int status = 0;
    *valid = 0;
    *best_iter = -1;
    *num_inliers = 0;
    *best_cost = 0.0f;
    if (n < 8) return 0;  /* H: min_set_size * 2; F: min_set_size */
    float* nk1 = (float*)malloc(sizeof(float) * 2 * (size_t)n1);
    float* nk2 = (float*)malloc(sizeof(float) * 2 * (size_t)n2);
    int32_t* idx = (int32_t*)malloc(sizeof(int32_t) * (size_t)n);
    double* S = (double*)malloc(sizeof(double) * 18 * (size_t)n);
    uint8_t* fl_sac = (uint8_t*)malloc((size_t)n);
    float mean[2], l1[2];
    double T1[9], T2[9], D2[9];
    orc_normalize(n1, kp1, nk1, mean, l1, T1);
    orc_normalize(n2, kp2, nk2, mean, l1, T2);
    tv_left_factor(model, T2, D2);
    float best = FLT_MAX;
    double bestM[9];
    memset(flags, 0, (size_t)n);
    for (int it = 0; it < n_iter; ++it) {
        double Mn[9], M[9];
        if (!tv_estimate(model, nk1, nk2, matches, min_sets + (size_t)set_size * it, set_size, S, Mn, &status)) continue;
        tv_denormalise(D2, Mn, T1, M);
        float cost;
        const unsigned num = tv_check_inliers(model, kp1, kp2, matches, n, M, sigma, fl_sac, &cost);
        if (num > (unsigned)set_size && best > cost) {
            best = cost;
            memcpy(bestM, M, sizeof bestM);
            memcpy(flags, fl_sac, (size_t)n);
            *best_iter = it;
            *num_inliers = (int)num;
        }
    }
    *best_cost = best;
    *valid = best < FLT_MAX;
    if (*valid && recompute) {
        int m = 0;
        for (int j = 0; j < n; ++j)
            if (flags[j]) idx[m++] = j;
        double Mn[9];
        if (tv_estimate(model, nk1, nk2, matches, idx, m, S, Mn, &status)) {
            tv_denormalise(D2, Mn, T1, bestM);
            tv_check_inliers(model, kp1, kp2, matches, n, bestM, sigma, flags, best_cost);
        }
    }
    if (*valid) memcpy(M_21, bestM, sizeof bestM);
    free(nk1);
    free(nk2);
    free(idx);
    free(S);
    free(fl_sac);
    return status;
}
