/* essential_oracle.c -- CPU restatement of solve::essential_solver::find_via_ransac (src/stella_vslam/solve/essential_solver.cc) with
 * the five-point minimal set.  The solver's arithmetic is stella_vslam_b200/csrc/essential_core.h compiled as C here
 * (-ffp-contract=off), on the SVD, Householder and util::cos pieces of tests/pnp_oracle.c (included, not copied); the RANSAC loop
 * below follows the reference's control flow directly.  The entry points also expose the stages (nullspace, constraint matrix,
 * eigen-decomposition, recompute) so the tests can check them against numpy / scipy.  Test infrastructure, compiled on first use. */
#include "pnp_oracle.c"

#include <stdlib.h>

#define ES_FN static
#define ES_BIG static
#define ES_SQRT(x) sqrt(x)
#define ES_MAKE_HOUSEHOLDER(v, len, stride, tau, beta) make_householder((v), (len), (stride), &(tau), &(beta))
#include "../stella_vslam_b200/csrc/essential_core.h"

/* find_nullspace_of_epipolar_constraint on five pairs (b1, b2: 5 x 3): basis 9 x 4 (row-major).  Returns 1 on success; *wide is 1
 * when the kernel had more than four columns. */
int orc_nullspace5(const double* b1, const double* b2, double* basis, int* wide) {
    const int32_t idx[5] = {0, 1, 2, 3, 4};
    int flags = 0;
    const int ok = es_nullspace5(b1, b2, idx, basis, &flags);
    *wide = (flags & ES_STATUS_WIDE_KER) != 0;
    return ok;
}

/* kernel() of a general n x n (n <= 9): K (n x n, first dimker columns).  Returns dimker. */
int orc_lu_kernel(int n, const double* A_in, double* K) {
    double A[81];
    int rowt[9], colt[9];
    double maxpivot;
    memcpy(A, A_in, sizeof(double) * n * n);
    const int nonzero = es_lu(n, A, rowt, colt, &maxpivot);
    return es_lu_kernel(n, A, colt, nonzero, maxpivot, K);
}

/* FullPivLU(A 10 x 10).solve(B 10 x 10).  Returns the rank. */
int orc_lu_solve10(const double* A_in, const double* B, double* X) {
    double A[100];
    int rowt[10], colt[10];
    double maxpivot;
    memcpy(A, A_in, sizeof A);
    const int nonzero = es_lu(10, A, rowt, colt, &maxpivot);
    es_lu_solve10(A, rowt, colt, nonzero, maxpivot, B, X);
    return es_lu_rank(10, A, nonzero, maxpivot);
}

void orc_constraint_matrix(const double* basis, double* M) { es_constraint_matrix(basis, M); }

/* EigenSolver<Mat10_t>: eigenvalues (re, im) and the real eigenvectors (columns of V).  Returns 0 or -1. */
int orc_eigen10(const double* A_in, double* re, double* im, double* V) {
    double A[100];
    memcpy(A, A_in, sizeof A);
    for (int k = 0; k < 100; ++k) V[k] = 0.0;
    return es_eigen(A, re, im, V);
}

/* compute_E_21_minimal on five pairs: up to ten row-major candidates.  Returns the count; *flags the ES_STATUS_* bits. */
int orc_minimal(const double* b1, const double* b2, double* E, int* flags) {
    const int32_t idx[5] = {0, 1, 2, 3, 4};
    *flags = 0;
    return es_minimal(b1, b2, idx, E, flags);
}

/* compute_E_21_nonminimal over m pairs.  Returns 0 or ES_STATUS_SVD. */
int orc_nonminimal(int m, const double* b1, const double* b2, double* E) {
    int32_t* idx = (int32_t*)malloc(sizeof(int32_t) * (size_t)m);
    double* S = (double*)malloc(sizeof(double) * 9 * (size_t)m);
    for (int i = 0; i < m; ++i) idx[i] = i;
    const int st = es_nonminimal(b1, b2, idx, m, S, E);
    free(idx);
    free(S);
    return st;
}

unsigned orc_check_inliers(int n, const double* b1, const double* b2, const double* E, uint8_t* flags, float* cost) {
    return es_check_inliers(b1, b2, n, E, es_cos_angle_thr(), flags, cost);
}

float orc_cos_angle_thr(void) { return es_cos_angle_thr(); }

/* find_via_ransac(max_num_iter = n_iter, recompute, 5) on the given minimal sets (n_iter x 5).  Outputs as b200_essential_problem_t;
 * flags untouched when n < 5.  Returns the status bits (ES_STATUS_SCHUR | ES_STATUS_SVD | ES_STATUS_WIDE_KER). */
int orc_essential_ransac(int n, const double* b1, const double* b2, int n_iter, int recompute, const int32_t* min_sets, int* valid,
                         int* best_iter, int* best_candidate, int* num_inliers, float* best_cost, double* E_21, uint8_t* flags) {
    int status = 0;
    *valid = 0;
    *best_iter = -1;
    *best_candidate = -1;
    *num_inliers = 0;
    *best_cost = 0.0f;
    if (n < 5) return 0;
    const float thr = es_cos_angle_thr();
    float best = FLT_MAX;
    double E[90], bestE[9];
    for (int it = 0; it < n_iter; ++it) {
        const int count = es_minimal(b1, b2, min_sets + 5 * (size_t)it, E, &status);
        for (int k = 0; k < count; ++k) {
            float cost;
            const unsigned num = es_check_inliers(b1, b2, n, E + 9 * k, thr, NULL, &cost);
            if (num > 5u && best > cost) {
                best = cost;
                memcpy(bestE, E + 9 * k, sizeof bestE);
                *best_iter = it;
                *best_candidate = k;
                *num_inliers = (int)num;
            }
        }
    }
    *best_cost = best;
    *valid = best < FLT_MAX;
    if (!*valid) {
        memset(flags, 0, (size_t)n);
        return status;
    }
    es_check_inliers(b1, b2, n, bestE, thr, flags, best_cost);
    *best_cost = best;
    if (recompute && *num_inliers >= 8) {
        int32_t* idx = (int32_t*)malloc(sizeof(int32_t) * (size_t)n);
        double* S = (double*)malloc(sizeof(double) * 9 * (size_t)n);
        int m = 0;
        for (int j = 0; j < n; ++j)
            if (flags[j]) idx[m++] = j;
        status |= es_nonminimal(b1, b2, idx, m, S, bestE);
        es_check_inliers(b1, b2, n, bestE, thr, flags, best_cost);
        free(idx);
        free(S);
    }
    memcpy(E_21, bestE, sizeof bestE);
    return status;
}
