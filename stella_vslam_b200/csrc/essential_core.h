/* essential_core.h -- solve::essential_solver (src/stella_vslam/solve/essential_solver.cc, essential_5pt.h): the five-point minimal
 * solver, check_inliers and the eight-point recompute, with the pieces of Eigen 3.4 they use restated from its algorithms:
 *   FullPivLU (full pivoting, first maximum in column-major order; rank() at |max pivot| * size * eps; kernel(); solve(), including
 *     the rank-deficient solve);
 *   EigenSolver: HessenbergDecomposition (Householder), RealSchur (Francis double shift, exceptional shifts at iterations 10 and 30,
 *     40 iterations per row in total), the eigenvalues, and the eigenvectors of the real eigenvalues only (back substitution through
 *     the quasi-triangular T, back transformation by Z, normalisation);
 *   JacobiSVD of the n x 9 eight-point matrix with ComputeFullV: wide (n = 8: ColPivHouseholderQR of the adjoint, V = its full Q),
 *     square (n = 9) and tall (n >= 10: ColPivHouseholderQR, V = its column permutation), then the 3 x 3 JacobiSVD.
 *
 * One source, compiled twice: as device code by essential_kernels.cu (explicit round-to-nearest intrinsics) and as C by
 * tests/essential_oracle.c (-ffp-contract=off), so the oracle computes every operation in the same order.  The includer defines
 *   ES_FN, ES_BIG                                  the function qualifiers (ES_BIG: the stages kept out of line, so
 *                                                  their work arrays do not add up in one stack frame);
 *   ES_SQRT(x)                                     a correctly rounded square root;
 *   ES_MAKE_HOUSEHOLDER(v, len, stride, tau, beta) makeHouseholderInPlace (tau, beta are lvalues);
 * and provides da / ds / dm / dd, svd_core, apply_householder_left and util_cos (epnp.cuh, util_trig.cuh / tests/pnp_oracle.c).
 * Sums run left to right in index order; Eigen's vectorised reductions and blocked triangular solves are not reproduced.
 * Matrices are row-major. */

/* ---- FullPivLU -------------------------------------------------------------------------------------------------------------- */

/* computeInPlace on the n x n A.  rowt / colt: the transpositions.  Returns the number of nonzero pivots; *maxpivot is m_maxpivot. */
ES_FN int es_lu(int n, double* A, int* rowt, int* colt, double* maxpivot) {
    int nonzero = n;
    *maxpivot = 0.0;
    for (int k = 0; k < n; ++k) {
        double big = fabs(A[k * n + k]);
        int br = k, bc = k;
        for (int c = k; c < n; ++c)  /* maxCoeff(&row, &col): column-major scan, the first strict maximum */
            for (int r = k; r < n; ++r) {
                const double s = fabs(A[r * n + c]);
                if (s > big) {
                    big = s;
                    br = r;
                    bc = c;
                }
            }
        if (big == 0.0) {
            nonzero = k;
            for (int i = k; i < n; ++i) rowt[i] = colt[i] = i;
            break;
        }
        if (big > *maxpivot) *maxpivot = big;
        rowt[k] = br;
        colt[k] = bc;
        if (br != k)
            for (int c = 0; c < n; ++c) {
                const double t = A[k * n + c];
                A[k * n + c] = A[br * n + c];
                A[br * n + c] = t;
            }
        if (bc != k)
            for (int r = 0; r < n; ++r) {
                const double t = A[r * n + k];
                A[r * n + k] = A[r * n + bc];
                A[r * n + bc] = t;
            }
        for (int r = k + 1; r < n; ++r) A[r * n + k] = dd(A[r * n + k], A[k * n + k]);
        for (int c = k + 1; c < n; ++c)
            for (int r = k + 1; r < n; ++r) A[r * n + c] = ds(A[r * n + c], dm(A[r * n + k], A[k * n + c]));
    }
    return nonzero;
}

ES_FN double es_lu_threshold(int n, double maxpivot) { return dm(fabs(maxpivot), dm((double)n, DBL_EPSILON)); }

ES_FN int es_lu_rank(int n, const double* A, int nonzero, double maxpivot) {
    const double thr = es_lu_threshold(n, maxpivot);
    int rank = 0;
    for (int i = 0; i < nonzero; ++i) rank += fabs(A[i * n + i]) > thr;
    return rank;
}

/* permutationQ().indices(): the identity with the column transpositions applied in order */
ES_FN void es_lu_q(int n, const int* colt, int* q) {
    for (int i = 0; i < n; ++i) q[i] = i;
    for (int k = 0; k < n; ++k) {
        const int t = q[k];
        q[k] = q[colt[k]];
        q[colt[k]] = t;
    }
}

/* triangularView<Upper>().solveInPlace on the rank x cols block at column c0 of the rank x ld matrix M (column-oriented, the
 * reciprocal of the pivot multiplied in, as Eigen's triangular_solve_matrix does) */
ES_FN void es_upper_solve(const double* U, int ldu, int rank, double* B, int ldb, int c0, int cols) {
    for (int j = c0; j < c0 + cols; ++j)
        for (int i = rank - 1; i >= 0; --i) {
            const double b = dm(B[i * ldb + j], dd(1.0, U[i * ldu + i]));
            B[i * ldb + j] = b;
            for (int r = 0; r < i; ++r) B[r * ldb + j] = ds(B[r * ldb + j], dm(b, U[r * ldu + i]));
        }
}

/* kernel() of the decomposed n x n (n <= 9): K (n x n, columns 0 .. dimker-1 written).  Returns dimker. */
ES_BIG int es_lu_kernel(int n, const double* A, const int* colt, int nonzero, double maxpivot, double* K) {
    const int rank = es_lu_rank(n, A, nonzero, maxpivot), dimker = n - rank;
    if (dimker == 0) return 0;
    const double thr = es_lu_threshold(n, maxpivot);
    int piv[9], q[9];
    double m[81];
    int p = 0;
    for (int i = 0; i < nonzero; ++i)
        if (fabs(A[i * n + i]) > thr) piv[p++] = i;
    for (int i = 0; i < rank; ++i)
        for (int c = 0; c < n; ++c) m[i * n + c] = c < i ? 0.0 : A[piv[i] * n + c];
    for (int i = 0; i < rank; ++i)
        if (piv[i] != i)
            for (int r = 0; r < rank; ++r) {
                const double t = m[r * n + i];
                m[r * n + i] = m[r * n + piv[i]];
                m[r * n + piv[i]] = t;
            }
    es_upper_solve(m, n, rank, m, n, rank, dimker);
    for (int i = rank - 1; i >= 0; --i)
        if (piv[i] != i)
            for (int r = 0; r < rank; ++r) {
                const double t = m[r * n + i];
                m[r * n + i] = m[r * n + piv[i]];
                m[r * n + piv[i]] = t;
            }
    es_lu_q(n, colt, q);
    for (int i = 0; i < rank; ++i)
        for (int k = 0; k < dimker; ++k) K[q[i] * n + k] = -m[i * n + rank + k];
    for (int i = rank; i < n; ++i)
        for (int k = 0; k < dimker; ++k) K[q[i] * n + k] = 0.0;
    for (int k = 0; k < dimker; ++k) K[q[rank + k] * n + k] = 1.0;
    return dimker;
}

/* solve() of the decomposed 10 x 10 against the 10 x 10 B: X */
ES_BIG void es_lu_solve10(const double* A, const int* rowt, const int* colt, int nonzero, double maxpivot, const double* B, double* X) {
    const int n = 10, rank = es_lu_rank(n, A, nonzero, maxpivot);
    if (rank == 0) {
        for (int k = 0; k < 100; ++k) X[k] = 0.0;
        return;
    }
    double c[100];
    int q[10];
    for (int k = 0; k < 100; ++k) c[k] = B[k];
    for (int k = 0; k < n; ++k)  /* permutationP() * rhs: the row transpositions in order */
        if (rowt[k] != k)
            for (int j = 0; j < n; ++j) {
                const double t = c[k * n + j];
                c[k * n + j] = c[rowt[k] * n + j];
                c[rowt[k] * n + j] = t;
            }
    for (int j = 0; j < n; ++j)  /* unit lower */
        for (int i = 0; i < n; ++i) {
            const double b = c[i * n + j];
            for (int r = i + 1; r < n; ++r) c[r * n + j] = ds(c[r * n + j], dm(b, A[r * n + i]));
        }
    es_upper_solve(A, n, rank, c, n, 0, n);
    es_lu_q(n, colt, q);
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) X[q[i] * n + j] = i < rank ? c[i * n + j] : 0.0;
}

/* ---- polynomial constraint matrix (essential_5pt.h) ------------------------------------------------------------------------- */

enum { ES_XXX, ES_XXY, ES_XYY, ES_YYY, ES_XXZ, ES_XYZ, ES_YYZ, ES_XZZ, ES_YZZ, ES_ZZZ, ES_XX, ES_XY, ES_YY, ES_XZ, ES_YZ, ES_ZZ, ES_X, ES_Y,
       ES_Z, ES_1 };

ES_FN void es_deg_one(const double* a, const double* b, double* p) {
    for (int k = 0; k < 20; ++k) p[k] = 0.0;
    p[ES_XX] = dm(a[ES_X], b[ES_X]);
    p[ES_XY] = da(dm(a[ES_X], b[ES_Y]), dm(a[ES_Y], b[ES_X]));
    p[ES_XZ] = da(dm(a[ES_X], b[ES_Z]), dm(a[ES_Z], b[ES_X]));
    p[ES_YY] = dm(a[ES_Y], b[ES_Y]);
    p[ES_YZ] = da(dm(a[ES_Y], b[ES_Z]), dm(a[ES_Z], b[ES_Y]));
    p[ES_ZZ] = dm(a[ES_Z], b[ES_Z]);
    p[ES_X] = da(dm(a[ES_X], b[ES_1]), dm(a[ES_1], b[ES_X]));
    p[ES_Y] = da(dm(a[ES_Y], b[ES_1]), dm(a[ES_1], b[ES_Y]));
    p[ES_Z] = da(dm(a[ES_Z], b[ES_1]), dm(a[ES_1], b[ES_Z]));
    p[ES_1] = dm(a[ES_1], b[ES_1]);
}

ES_FN void es_deg_two(const double* a, const double* b, double* p) {
    p[ES_XXX] = dm(a[ES_XX], b[ES_X]);
    p[ES_XXY] = da(dm(a[ES_XX], b[ES_Y]), dm(a[ES_XY], b[ES_X]));
    p[ES_XXZ] = da(dm(a[ES_XX], b[ES_Z]), dm(a[ES_XZ], b[ES_X]));
    p[ES_XYY] = da(dm(a[ES_XY], b[ES_Y]), dm(a[ES_YY], b[ES_X]));
    p[ES_XYZ] = da(da(dm(a[ES_XY], b[ES_Z]), dm(a[ES_YZ], b[ES_X])), dm(a[ES_XZ], b[ES_Y]));
    p[ES_XZZ] = da(dm(a[ES_XZ], b[ES_Z]), dm(a[ES_ZZ], b[ES_X]));
    p[ES_YYY] = dm(a[ES_YY], b[ES_Y]);
    p[ES_YYZ] = da(dm(a[ES_YY], b[ES_Z]), dm(a[ES_YZ], b[ES_Y]));
    p[ES_YZZ] = da(dm(a[ES_YZ], b[ES_Z]), dm(a[ES_ZZ], b[ES_Y]));
    p[ES_ZZZ] = dm(a[ES_ZZ], b[ES_Z]);
    p[ES_XX] = da(dm(a[ES_XX], b[ES_1]), dm(a[ES_X], b[ES_X]));
    p[ES_XY] = da(da(dm(a[ES_XY], b[ES_1]), dm(a[ES_X], b[ES_Y])), dm(a[ES_Y], b[ES_X]));
    p[ES_XZ] = da(da(dm(a[ES_XZ], b[ES_1]), dm(a[ES_X], b[ES_Z])), dm(a[ES_Z], b[ES_X]));
    p[ES_YY] = da(dm(a[ES_YY], b[ES_1]), dm(a[ES_Y], b[ES_Y]));
    p[ES_YZ] = da(da(dm(a[ES_YZ], b[ES_1]), dm(a[ES_Y], b[ES_Z])), dm(a[ES_Z], b[ES_Y]));
    p[ES_ZZ] = da(dm(a[ES_ZZ], b[ES_1]), dm(a[ES_Z], b[ES_Z]));
    p[ES_X] = da(dm(a[ES_X], b[ES_1]), dm(a[ES_1], b[ES_X]));
    p[ES_Y] = da(dm(a[ES_Y], b[ES_1]), dm(a[ES_1], b[ES_Y]));
    p[ES_Z] = da(dm(a[ES_Z], b[ES_1]), dm(a[ES_1], b[ES_Z]));
    p[ES_1] = dm(a[ES_1], b[ES_1]);
}

/* d1(a0, b0) - d1(a1, b1) */
ES_FN void es_deg_one_diff(const double* a0, const double* b0, const double* a1, const double* b1, double* p) {
    double u[20], v[20];
    es_deg_one(a0, b0, u);
    es_deg_one(a1, b1, v);
    for (int k = 0; k < 20; ++k) p[k] = ds(u[k], v[k]);
}

/* form_polynomial_constraint_matrix: basis is 9 x 4 (row-major), M is 10 x 20 */
ES_BIG void es_constraint_matrix(const double* basis, double* M) {
    double E[3][3][20], EET[3][3][20];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            for (int k = 0; k < 20; ++k) E[i][j][k] = 0.0;
            E[i][j][ES_X] = basis[(3 * i + j) * 4 + 0];
            E[i][j][ES_Y] = basis[(3 * i + j) * 4 + 1];
            E[i][j][ES_Z] = basis[(3 * i + j) * 4 + 2];
            E[i][j][ES_1] = basis[(3 * i + j) * 4 + 3];
        }
    {
        double d[20], t0[20], t1[20], t2[20];
        es_deg_one_diff(E[0][1], E[1][2], E[0][2], E[1][1], d);
        es_deg_two(d, E[2][0], t0);
        es_deg_one_diff(E[0][2], E[1][0], E[0][0], E[1][2], d);
        es_deg_two(d, E[2][1], t1);
        es_deg_one_diff(E[0][0], E[1][1], E[0][1], E[1][0], d);
        es_deg_two(d, E[2][2], t2);
        for (int k = 0; k < 20; ++k) M[k] = da(da(t0[k], t1[k]), t2[k]);
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            if (i <= j) {
                double u[20], v[20], w[20];
                es_deg_one(E[i][0], E[j][0], u);
                es_deg_one(E[i][1], E[j][1], v);
                es_deg_one(E[i][2], E[j][2], w);
                for (int k = 0; k < 20; ++k) EET[i][j][k] = da(da(u[k], v[k]), w[k]);
            } else {
                for (int k = 0; k < 20; ++k) EET[i][j][k] = EET[j][i][k];
            }
        }
    double trace[20];
    for (int k = 0; k < 20; ++k) trace[k] = dm(0.5, da(da(EET[0][0][k], EET[1][1][k]), EET[2][2][k]));
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 20; ++k) EET[i][i][k] = ds(EET[i][i][k], trace[k]);
    int row = 1;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double t0[20], t1[20], t2[20];
            es_deg_two(EET[i][0], E[0][j], t0);
            es_deg_two(EET[i][1], E[1][j], t1);
            es_deg_two(EET[i][2], E[2][j], t2);
            for (int k = 0; k < 20; ++k) M[row * 20 + k] = da(da(t0[k], t1[k]), t2[k]);
            ++row;
        }
}

/* ---- EigenSolver<Mat10_t> --------------------------------------------------------------------------------------------------- */

/* applyHouseholderOnTheRight to the block B (rows x cols, row stride ldb) with the essential part ess[0..cols-2] (stride es) */
ES_FN void es_householder_right(double* B, int rows, int cols, int ldb, const double* ess, int es, double tau) {
    if (cols == 1) {
        const double f = ds(1.0, tau);
        for (int r = 0; r < rows; ++r) B[r * ldb] = dm(B[r * ldb], f);
        return;
    }
    if (tau == 0.0) return;
    for (int r = 0; r < rows; ++r) {
        double* row = &B[r * ldb];
        double tmp = dm(row[1], ess[0]);
        for (int j = 1; j < cols - 1; ++j) tmp = da(tmp, dm(row[1 + j], ess[j * es]));
        tmp = da(tmp, row[0]);
        const double tt = dm(tau, tmp);
        row[0] = ds(row[0], tt);
        for (int j = 0; j < cols - 1; ++j) row[1 + j] = ds(row[1 + j], dm(tt, ess[j * es]));
    }
}

/* rows p, q of B (columns c0 .. c1-1, stride 1) and columns p, q (rows r0 .. r1-1) by the rotation (c, s), as apply_rotation_in_the_plane */
ES_FN void es_rot_rows(double* T, int p, int q, int c0, int c1, double c, double s) {
    for (int k = c0; k < c1; ++k) {
        const double xi = T[p * 10 + k], yi = T[q * 10 + k];
        T[p * 10 + k] = da(dm(c, xi), dm(s, yi));
        T[q * 10 + k] = da(dm(-s, xi), dm(c, yi));
    }
}
ES_FN void es_rot_cols(double* T, int p, int q, int r0, int r1, double c, double s) {
    for (int k = r0; k < r1; ++k) {
        const double xi = T[k * 10 + p], yi = T[k * 10 + q];
        T[k * 10 + p] = da(dm(c, xi), dm(s, yi));
        T[k * 10 + q] = da(dm(-s, xi), dm(c, yi));
    }
}

/* JacobiRotation::makeGivens(p, q) */
ES_FN void es_make_givens(double p, double q, double* c, double* s) {
    if (q == 0.0) {
        *c = p < 0.0 ? -1.0 : 1.0;
        *s = 0.0;
    } else if (p == 0.0) {
        *c = 0.0;
        *s = q < 0.0 ? 1.0 : -1.0;
    } else if (fabs(p) > fabs(q)) {
        const double t = dd(q, p);
        double u = ES_SQRT(da(1.0, dm(t, t)));
        if (p < 0.0) u = -u;
        *c = dd(1.0, u);
        *s = dm(-t, *c);
    } else {
        const double t = dd(p, q);
        double u = ES_SQRT(da(1.0, dm(t, t)));
        if (q < 0.0) u = -u;
        *s = dd(-1.0, u);
        *c = dm(-t, *s);
    }
}

ES_FN double es_max(double a, double b) { return a < b ? b : a; }

/* RealSchur<Mat10_t>::compute(A, true): T (in: A, out: the quasi-triangular T), U.  Returns 0, or -1 when it did not converge. */
ES_BIG int es_real_schur(double* T, double* U) {
    const int n = 10;
    double scale = 0.0;
    for (int k = 0; k < 100; ++k) scale = es_max(scale, fabs(T[k]));
    if (scale < DBL_MIN) {
        for (int k = 0; k < 100; ++k) {
            T[k] = 0.0;
            U[k] = (k % 11 == 0) ? 1.0 : 0.0;
        }
        return 0;
    }
    for (int k = 0; k < 100; ++k) T[k] = dd(T[k], scale);
    /* HessenbergDecomposition: the Householder vectors stay below the subdiagonal until Q is formed */
    double hc[9];
    for (int i = 0; i < n - 1; ++i) {
        const int rem = n - i - 1;
        double h, beta;
        ES_MAKE_HOUSEHOLDER(&T[(i + 1) * n + i], rem, n, h, beta);
        T[(i + 1) * n + i] = beta;
        hc[i] = h;
        apply_householder_left(&T[(i + 1) * n + i + 1], rem, rem, n, &T[(i + 2) * n + i], n, h);
        es_householder_right(&T[i + 1], n, rem, n, &T[(i + 2) * n + i], n, h);
    }
    for (int k = 0; k < 100; ++k) U[k] = (k % 11 == 0) ? 1.0 : 0.0;
    for (int k = n - 2; k >= 0; --k) {
        const int cs = n - k - 1;
        apply_householder_left(&U[(k + 1) * n + k + 1], cs, cs, n, &T[(k + 2) * n + k], n, hc[k]);
    }
    for (int r = 2; r < n; ++r)
        for (int c = 0; c < r - 1; ++c) T[r * n + c] = 0.0;

    /* computeFromHessenberg */
    int iu = n - 1, iter = 0, total_iter = 0;
    const int max_iters = 40 * n;
    double exshift = 0.0;
    double norm = 0.0;
    for (int j = 0; j < n; ++j) {
        const int len = j + 2 < n ? j + 2 : n;
        double s = fabs(T[j]);
        for (int i = 1; i < len; ++i) s = da(s, fabs(T[i * n + j]));
        norm = da(norm, s);
    }
    const double consider_as_zero = es_max(dm(norm, dm(DBL_EPSILON, DBL_EPSILON)), DBL_MIN);
    if (norm != 0.0) {
        while (iu >= 0) {
            int il = iu;
            while (il > 0) {
                double s = da(fabs(T[(il - 1) * n + il - 1]), fabs(T[il * n + il]));
                s = es_max(dm(s, DBL_EPSILON), consider_as_zero);
                if (fabs(T[il * n + il - 1]) <= s) break;
                --il;
            }
            if (il == iu) {
                T[iu * n + iu] = da(T[iu * n + iu], exshift);
                if (iu > 0) T[iu * n + iu - 1] = 0.0;
                --iu;
                iter = 0;
            } else if (il == iu - 1) {
                const double p = dm(0.5, ds(T[(iu - 1) * n + iu - 1], T[iu * n + iu]));
                const double q = da(dm(p, p), dm(T[iu * n + iu - 1], T[(iu - 1) * n + iu]));
                T[iu * n + iu] = da(T[iu * n + iu], exshift);
                T[(iu - 1) * n + iu - 1] = da(T[(iu - 1) * n + iu - 1], exshift);
                if (q >= 0.0) {
                    const double z = ES_SQRT(fabs(q));
                    double c, s;
                    es_make_givens(p >= 0.0 ? da(p, z) : ds(p, z), T[iu * n + iu - 1], &c, &s);
                    es_rot_rows(T, iu - 1, iu, iu - 1, n, c, -s);
                    es_rot_cols(T, iu - 1, iu, 0, iu + 1, c, -s);
                    T[iu * n + iu - 1] = 0.0;
                    es_rot_cols(U, iu - 1, iu, 0, n, c, -s);
                }
                if (iu > 1) T[(iu - 1) * n + iu - 2] = 0.0;
                iu -= 2;
                iter = 0;
            } else {
                /* computeShift */
                double sh0 = T[iu * n + iu], sh1 = T[(iu - 1) * n + iu - 1], sh2 = dm(T[iu * n + iu - 1], T[(iu - 1) * n + iu]);
                if (iter == 10) {
                    exshift = da(exshift, sh0);
                    for (int i = 0; i <= iu; ++i) T[i * n + i] = ds(T[i * n + i], sh0);
                    const double s = da(fabs(T[iu * n + iu - 1]), fabs(T[(iu - 1) * n + iu - 2]));
                    sh0 = dm(0.75, s);
                    sh1 = dm(0.75, s);
                    sh2 = dm(dm(-0.4375, s), s);
                }
                if (iter == 30) {
                    double s = dd(ds(sh1, sh0), 2.0);
                    s = da(dm(s, s), sh2);
                    if (s > 0.0) {
                        s = ES_SQRT(s);
                        if (sh1 < sh0) s = -s;
                        s = da(s, dd(ds(sh1, sh0), 2.0));
                        s = ds(sh0, dd(sh2, s));
                        exshift = da(exshift, s);
                        for (int i = 0; i <= iu; ++i) T[i * n + i] = ds(T[i * n + i], s);
                        sh0 = sh1 = sh2 = 0.964;
                    }
                }
                ++iter;
                ++total_iter;
                if (total_iter > max_iters) break;
                /* initFrancisQRStep */
                double v[3] = {0.0, 0.0, 0.0};
                int im;
                for (im = iu - 2; im >= il; --im) {
                    const double Tmm = T[im * n + im];
                    const double r = ds(sh0, Tmm), s = ds(sh1, Tmm);
                    v[0] = da(dd(ds(dm(r, s), sh2), T[(im + 1) * n + im]), T[im * n + im + 1]);
                    v[1] = ds(ds(ds(T[(im + 1) * n + im + 1], Tmm), r), s);
                    v[2] = T[(im + 2) * n + im + 1];
                    if (im == il) break;
                    const double lhs = dm(T[im * n + im - 1], da(fabs(v[1]), fabs(v[2])));
                    const double rhs = dm(v[0], da(da(fabs(T[(im - 1) * n + im - 1]), fabs(Tmm)), fabs(T[(im + 1) * n + im + 1])));
                    if (fabs(lhs) < dm(DBL_EPSILON, rhs)) break;
                }
                /* performFrancisQRStep */
                for (int k = im; k <= iu - 2; ++k) {
                    const int first = k == im;
                    double w[3];
                    if (first) {
                        w[0] = v[0];
                        w[1] = v[1];
                        w[2] = v[2];
                    } else {
                        w[0] = T[k * n + k - 1];
                        w[1] = T[(k + 1) * n + k - 1];
                        w[2] = T[(k + 2) * n + k - 1];
                    }
                    double tau, beta;
                    ES_MAKE_HOUSEHOLDER(w, 3, 1, tau, beta);
                    if (beta != 0.0) {
                        if (first && k > il)
                            T[k * n + k - 1] = -T[k * n + k - 1];
                        else if (!first)
                            T[k * n + k - 1] = beta;
                        apply_householder_left(&T[k * n + k], 3, n - k, n, &w[1], 1, tau);
                        es_householder_right(&T[k], (iu < k + 3 ? iu : k + 3) + 1, 3, n, &w[1], 1, tau);
                        es_householder_right(&U[k], n, 3, n, &w[1], 1, tau);
                    }
                }
                {
                    double w[2] = {T[(iu - 1) * n + iu - 2], T[iu * n + iu - 2]};
                    double tau, beta;
                    ES_MAKE_HOUSEHOLDER(w, 2, 1, tau, beta);
                    if (beta != 0.0) {
                        T[(iu - 1) * n + iu - 2] = beta;
                        apply_householder_left(&T[(iu - 1) * n + iu - 1], 2, n - iu + 1, n, &w[1], 1, tau);
                        es_householder_right(&T[iu - 1], iu + 1, 2, n, &w[1], 1, tau);
                        es_householder_right(&U[iu - 1], n, 2, n, &w[1], 1, tau);
                    }
                }
                for (int i = im + 2; i <= iu; ++i) {
                    T[i * n + i - 2] = 0.0;
                    if (i > im + 2) T[i * n + i - 3] = 0.0;
                }
            }
        }
    }
    if (total_iter > max_iters) return -1;
    for (int k = 0; k < 100; ++k) T[k] = dm(T[k], scale);
    return 0;
}

/* EigenSolver<Mat10_t>(A): the eigenvalues (re, im) and, for every eigenvalue with im == 0, the normalised real eigenvector in
 * column s of V (10 x 10).  A is overwritten.  Returns 0, or -1 when RealSchur did not converge or an eigenvalue is not finite. */
ES_BIG int es_eigen(double* A, double* re, double* im, double* V) {
    const int n = 10;
    double U[100];
    if (es_real_schur(A, U) < 0) return -1;
    double* T = A;
    for (int i = 0; i < n;) {
        if (i == n - 1 || T[(i + 1) * n + i] == 0.0) {
            re[i] = T[i * n + i];
            im[i] = 0.0;
            if (!isfinite(re[i])) return -1;
            ++i;
        } else {
            const double p = dm(0.5, ds(T[i * n + i], T[(i + 1) * n + i + 1]));
            double t0 = T[(i + 1) * n + i], t1 = T[i * n + i + 1];
            const double maxval = es_max(fabs(p), es_max(fabs(t0), fabs(t1)));
            t0 = dd(t0, maxval);
            t1 = dd(t1, maxval);
            const double p0 = dd(p, maxval);
            const double z = dm(maxval, ES_SQRT(fabs(da(dm(p0, p0), dm(t0, t1)))));
            re[i] = re[i + 1] = da(T[(i + 1) * n + i + 1], p);
            im[i] = z;
            im[i + 1] = -z;
            if (!(isfinite(re[i]) && isfinite(z))) return -1;
            i += 2;
        }
    }
    /* doComputeEigenvectors, real eigenvalues only: a complex pair writes only its own two columns of T, which no real column left of
     * them reads */
    double norm = 0.0;
    for (int j = 0; j < n; ++j) {
        const int c0 = j - 1 > 0 ? j - 1 : 0;
        double s = fabs(T[j * n + c0]);
        for (int c = c0 + 1; c < n; ++c) s = da(s, fabs(T[j * n + c]));
        norm = da(norm, s);
    }
    for (int s = n - 1; s >= 0; --s) {  /* descending, as Eigen: column s reads the columns left of it unmodified */
        if (im[s] != 0.0) continue;
        double v[10];
        if (norm == 0.0) {
            for (int r = 0; r < n; ++r) v[r] = U[r * n + s];
        } else {
            const double p = re[s];
            double lastr = 0.0, lastw = 0.0;
            int l = s;
            T[s * n + s] = 1.0;
            for (int i = s - 1; i >= 0; --i) {
                const double w = ds(T[i * n + i], p);
                double r = dm(T[i * n + l], T[l * n + s]);
                for (int c = l + 1; c <= s; ++c) r = da(r, dm(T[i * n + c], T[c * n + s]));
                if (im[i] < 0.0) {
                    lastw = w;
                    lastr = r;
                } else {
                    l = i;
                    if (im[i] == 0.0) {
                        T[i * n + s] = w != 0.0 ? dd(-r, w) : dd(-r, dm(DBL_EPSILON, norm));
                    } else {
                        const double x = T[i * n + i + 1], y = T[(i + 1) * n + i];
                        const double dr = ds(re[i], p);
                        const double denom = da(dm(dr, dr), dm(im[i], im[i]));
                        const double t = dd(ds(dm(x, lastr), dm(lastw, r)), denom);
                        T[i * n + s] = t;
                        if (fabs(x) > fabs(lastw))
                            T[(i + 1) * n + s] = dd(ds(-r, dm(w, t)), x);
                        else
                            T[(i + 1) * n + s] = dd(ds(-lastr, dm(y, t)), lastw);
                    }
                    const double t = fabs(T[i * n + s]);
                    if (dm(dm(DBL_EPSILON, t), t) > 1.0)
                        for (int r2 = i; r2 < n; ++r2) T[r2 * n + s] = dd(T[r2 * n + s], t);
                }
            }
            for (int r = 0; r < n; ++r) {  /* m_eivec.leftCols(s + 1) * T.col(s).head(s + 1) */
                double a = dm(U[r * n], T[s]);
                for (int k = 1; k <= s; ++k) a = da(a, dm(U[r * n + k], T[k * n + s]));
                v[r] = a;
            }
        }
        double z = dm(v[0], v[0]);
        for (int r = 1; r < n; ++r) z = da(z, dm(v[r], v[r]));
        if (z > 0.0) {
            const double sq = ES_SQRT(z);
            for (int r = 0; r < n; ++r) v[r] = dd(v[r], sq);
        }
        for (int r = 0; r < n; ++r) V[r * n + s] = v[r];
    }
    return 0;
}

/* ---- compute_E_21_minimal ----------------------------------------------------------------------------------------------------- */

#define ES_STATUS_SCHUR 1     /* RealSchur did not converge (or an eigenvalue is not finite): no candidates */
#define ES_STATUS_SVD 2       /* a Jacobi SVD of the recompute hit its sweep bound */
#define ES_STATUS_WIDE_KER 4  /* the five-point nullspace had more than four columns: the first four were used (EXT?) */

/* find_nullspace_of_epipolar_constraint (five pairs): the 9 x 4 basis.  Returns 1 on success (dimensionOfKernel() >= 4). */
ES_BIG int es_nullspace5(const double* b1, const double* b2, const int32_t* idx, double* basis, int* flags) {
    double A[81], K[81];
    int rowt[9], colt[9];
    for (int k = 0; k < 81; ++k) A[k] = 0.0;
    for (int i = 0; i < 5; ++i) {
        const double* x1 = b1 + 3 * (size_t)idx[i];
        const double* x2 = b2 + 3 * (size_t)idx[i];
        for (int a = 0; a < 3; ++a)
            for (int c = 0; c < 3; ++c) A[i * 9 + 3 * a + c] = dm(x2[a], x1[c]);
    }
    double maxpivot;
    const int nonzero = es_lu(9, A, rowt, colt, &maxpivot);
    const int dimker = es_lu_kernel(9, A, colt, nonzero, maxpivot, K);
    if (dimker < 4) return 0;
    if (dimker > 4) *flags |= ES_STATUS_WIDE_KER;
    for (int r = 0; r < 9; ++r)
        for (int k = 0; k < 4; ++k) basis[r * 4 + k] = K[r * 9 + k];
    return 1;
}

/* compute_E_21_minimal on the five pairs idx[0..4]: up to ten candidates (row-major E_21, in eigenvalue order) into E.
 * Returns the count; *flags gains ES_STATUS_* bits. */
ES_FN int es_minimal(const double* b1, const double* b2, const int32_t* idx, double* E, int* flags) {
    /* the stage arrays share one buffer (the thread's stack frame is the local-memory reservation of every resident thread):
     * M = w[0, 200), L = w[200, 300), R = w[300, 400); then X = w[0, 100) once M is split; then A = w[100, 200), V = w[200, 300) */
    double basis[36], w[400], re[10], im[10];
    if (!es_nullspace5(b1, b2, idx, basis, flags)) return 0;
    double* M = w;
    double* L = w + 200;
    double* R = w + 300;
    double* X = w;
    double* A = w + 100;
    double* V = w + 200;
    es_constraint_matrix(basis, M);
    {
        int rowt[10], colt[10];
        for (int r = 0; r < 10; ++r)
            for (int c = 0; c < 10; ++c) {
                L[r * 10 + c] = M[r * 20 + c];
                R[r * 10 + c] = M[r * 20 + 10 + c];
            }
        double maxpivot;
        const int nonzero = es_lu(10, L, rowt, colt, &maxpivot);
        es_lu_solve10(L, rowt, colt, nonzero, maxpivot, R, X);
    }
    for (int k = 0; k < 100; ++k) A[k] = 0.0;
    for (int c = 0; c < 10; ++c) {
        A[0 * 10 + c] = X[0 * 10 + c];
        A[1 * 10 + c] = X[1 * 10 + c];
        A[2 * 10 + c] = X[2 * 10 + c];
        A[3 * 10 + c] = X[4 * 10 + c];
        A[4 * 10 + c] = X[5 * 10 + c];
        A[5 * 10 + c] = X[7 * 10 + c];
    }
    A[6 * 10 + 0] = -1.0;
    A[7 * 10 + 1] = -1.0;
    A[8 * 10 + 3] = -1.0;
    A[9 * 10 + 6] = -1.0;
    if (es_eigen(A, re, im, V) < 0) {
        *flags |= ES_STATUS_SCHUR;
        return 0;
    }
    int count = 0;
    for (int s = 0; s < 10; ++s) {
        if (im[s] != 0.0) continue;
        double* e = E + 9 * count;
        for (int r = 0; r < 9; ++r) {  /* E_basis * eig_vecs.col(s).tail<4>(), then Mat33_t(data).transpose(): row-major */
            double a = dm(basis[r * 4], V[6 * 10 + s]);
            for (int k = 1; k < 4; ++k) a = da(a, dm(basis[r * 4 + k], V[(6 + k) * 10 + s]));
            e[r] = a;
        }
        ++count;
    }
    return count;
}

/* ---- check_inliers ------------------------------------------------------------------------------------------------------------ */

ES_FN float es_cos_angle_thr(void) { return util_cos((float)(1.0 * M_PI / 180.0)); }

/* |cross(e, b)| / |e| as float */
ES_FN float es_epi_cos(const double* e, const double* b) {
    const double c0 = ds(dm(e[1], b[2]), dm(e[2], b[1]));
    const double c1 = ds(dm(e[2], b[0]), dm(e[0], b[2]));
    const double c2 = ds(dm(e[0], b[1]), dm(e[1], b[0]));
    const double cn = ES_SQRT(da(da(dm(c0, c0), dm(c1, c1)), dm(c2, c2)));
    const double en = ES_SQRT(da(da(dm(e[0], e[0]), dm(e[1], e[1])), dm(e[2], e[2])));
    return (float)dd(cn, en);
}

/* check_inliers(E_21): the float cost accumulated in ascending match order; flags (may be null) receive the decisions */
ES_FN unsigned es_check_inliers(const double* b1, const double* b2, int n, const double* E, float thr, uint8_t* flags, float* cost) {
    unsigned num = 0;
    float c = 0.0f;
    for (int j = 0; j < n; ++j) {
        const double* x1 = b1 + 3 * (size_t)j;
        const double* x2 = b2 + 3 * (size_t)j;
        double e2[3], e1[3];
        for (int r = 0; r < 3; ++r) {
            e2[r] = da(da(dm(E[r * 3], x1[0]), dm(E[r * 3 + 1], x1[1])), dm(E[r * 3 + 2], x1[2]));
            e1[r] = da(da(dm(E[r], x2[0]), dm(E[3 + r], x2[1])), dm(E[6 + r], x2[2]));
        }
        const float cos_in_2 = es_epi_cos(e2, x2);
        const float cos_in_1 = es_epi_cos(e1, x1);
        const float worst = (cos_in_2 < cos_in_1) ? cos_in_2 : cos_in_1;  /* std::min: NaN in cos_in_1 propagates, in cos_in_2 does not */
        const int in = thr < worst;
        if (in) {
            c = (float)da((double)c, ds(1.0, (double)worst));
            ++num;
        } else {
            c = (float)da((double)c, ds(1.0, (double)thr));
        }
        if (flags) flags[j] = (uint8_t)in;
    }
    *cost = c;
    return num;
}

/* ---- compute_E_21_nonminimal ---------------------------------------------------------------------------------------------------- */

/* ColPivHouseholderQR of the rows x cols S (row-major, in place): htau, perm (colsPermutation().indices()) */
ES_BIG void es_colpiv_qr(int rows, int cols, double* S, double* htau, int* perm) {
    double cn_upd[9], cn_dir[9];
    for (int j = 0; j < cols; ++j) {
        double s = dm(S[j], S[j]);
        for (int i = 1; i < rows; ++i) s = da(s, dm(S[i * cols + j], S[i * cols + j]));
        cn_dir[j] = ES_SQRT(s);
        cn_upd[j] = cn_dir[j];
        perm[j] = j;
    }
    const double norm_downdate_threshold = ES_SQRT(DBL_EPSILON);
    const int size = rows < cols ? rows : cols;
    for (int c = 0; c < size; ++c) {
        int big = c;
        for (int j = c + 1; j < cols; ++j)
            if (cn_upd[j] > cn_upd[big]) big = j;
        if (big != c) {
            for (int i = 0; i < rows; ++i) {
                const double t = S[i * cols + c];
                S[i * cols + c] = S[i * cols + big];
                S[i * cols + big] = t;
            }
            double t = cn_upd[c];
            cn_upd[c] = cn_upd[big];
            cn_upd[big] = t;
            t = cn_dir[c];
            cn_dir[c] = cn_dir[big];
            cn_dir[big] = t;
            const int ti = perm[c];
            perm[c] = perm[big];
            perm[big] = ti;
        }
        double beta;
        ES_MAKE_HOUSEHOLDER(&S[c * cols + c], rows - c, cols, htau[c], beta);
        S[c * cols + c] = beta;
        if (cols - c - 1 > 0) apply_householder_left(&S[c * cols + c + 1], rows - c, cols - c - 1, cols, &S[(c + 1) * cols + c], cols, htau[c]);
        for (int j = c + 1; j < cols; ++j) {
            if (cn_upd[j] == 0.0) continue;
            double temp = dd(fabs(S[c * cols + j]), cn_upd[j]);
            temp = dm(da(1.0, temp), ds(1.0, temp));
            temp = temp < 0.0 ? 0.0 : temp;
            const double r = dd(cn_upd[j], cn_dir[j]);
            const double temp2 = dm(temp, dm(r, r));
            if (temp2 <= norm_downdate_threshold) {
                double s = 0.0;
                for (int i = c + 1; i < rows; ++i) s = (i == c + 1) ? dm(S[i * cols + j], S[i * cols + j]) : da(s, dm(S[i * cols + j], S[i * cols + j]));
                cn_dir[j] = ES_SQRT(s);
                cn_upd[j] = cn_dir[j];
            } else {
                cn_upd[j] = dm(cn_upd[j], ES_SQRT(temp));
            }
        }
    }
}

/* The singular values of the wide path's 8 x 8 work matrix, R^T of the adjoint's QR (At: 9 x 8 after es_colpiv_qr).  U and V are not
 * formed: the callers need neither.  Returns svd_core's count. */
ES_BIG int es_wide_sv(const double* At, double scale, double* sv) {
    double W[64];
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) W[i * 8 + j] = j <= i ? At[j * 8 + i] : 0.0;
    return svd_core(8, W, 0, NULL, NULL, scale, sv);
}

/* JacobiSVD<Matrix<double, Dynamic, 9>> (ComputeFullV) of the m x 9 S (row-major, m >= 8; overwritten on the tall path), scale its
 * max |entry| (1 when all are zero): V's last column into v9.  With sv non-null also the min(m, 9) singular values in descending order
 * and *nonzero, svd_core's count (m_nonzeroSingularValues; -1 when the sweeps hit their bound).  The wide path then also sweeps its
 * 8 x 8 work matrix, which V's last column does not depend on.  Returns 0, or ES_STATUS_SVD.
 *   wide (m = 8): ColPivHouseholderQR of the adjoint (9 x 8); V = its full Q, whose last column no sweep touches;
 *   square (m = 9): no preconditioner;
 *   tall (m >= 10): ColPivHouseholderQR; the work matrix is R, V the column permutation. */
ES_BIG int es_svd_n9(int m, double* S, double scale, double* v9, double* sv, int* nonzero) {
    int status = 0;
    if (m == 8) {
        double At[72], htau[8], Q[81];
        int perm[8];
        for (int i = 0; i < 8; ++i)
            for (int c = 0; c < 9; ++c) At[c * 8 + i] = dd(S[i * 9 + c], scale);
        es_colpiv_qr(9, 8, At, htau, perm);
        for (int k = 0; k < 81; ++k) Q[k] = (k % 10 == 0) ? 1.0 : 0.0;
        for (int c = 7; c >= 0; --c) apply_householder_left(&Q[c * 9 + c], 9 - c, 9 - c, 9, &At[(c + 1) * 8 + c], 8, htau[c]);
        for (int r = 0; r < 9; ++r) v9[r] = Q[r * 9 + 8];
        if (sv) {
            *nonzero = es_wide_sv(At, scale, sv);
            if (*nonzero < 0) status = ES_STATUS_SVD;
        }
    } else {
        double W[81], V[81], s9[9];
        if (m == 9) {
            for (int k = 0; k < 81; ++k) {
                W[k] = dd(S[k], scale);
                V[k] = (k % 10 == 0) ? 1.0 : 0.0;
            }
        } else {
            double htau[9];
            int perm[9];
            for (size_t k = 0; k < (size_t)m * 9; ++k) S[k] = dd(S[k], scale);
            es_colpiv_qr(m, 9, S, htau, perm);
            for (int i = 0; i < 9; ++i)
                for (int j = 0; j < 9; ++j) {
                    W[i * 9 + j] = j >= i ? S[i * 9 + j] : 0.0;
                    V[i * 9 + j] = (i == perm[j]) ? 1.0 : 0.0;
                }
        }
        const int nz = svd_core(9, W, 0, NULL, V, scale, s9);
        if (nz < 0) status = ES_STATUS_SVD;
        for (int r = 0; r < 9; ++r) v9[r] = V[r * 9 + 8];
        if (sv) {
            for (int k = 0; k < 9; ++k) sv[k] = s9[k];
            *nonzero = nz;
        }
    }
    return status;
}

/* JacobiSVD::rank() at its default threshold: the singular values >= max(s0 * diag * eps, DBL_MIN), counted down from the last
 * nonzero one (diag = min(rows, cols)).  A sweep that hit its bound (nonzero < 0) counts as rank 0. */
ES_FN int es_svd_rank(int diag, const double* sv, int nonzero) {
    if (nonzero <= 0) return 0;
    const double thr = es_max(dm(sv[0], dm((double)diag, DBL_EPSILON)), DBL_MIN);
    int i = nonzero - 1;
    while (i >= 0 && sv[i] < thr) --i;
    return i + 1;
}

/* Mat33_t(v.data()).transpose() (row-major v9), then JacobiSVD<Mat33_t>, lambda(2) = 0, U diag(lambda) V^T into E: the rank-2
 * projection shared by compute_E_21_nonminimal and fundamental_solver::compute_F_21.  Returns 0, or ES_STATUS_SVD. */
ES_BIG int es_rank2(const double* v9, double* E) {
    int status = 0;
    double W3[9], U3[9], V3[9], s3[3];
    double sc = 0.0;
    for (int k = 0; k < 9; ++k) sc = es_max(sc, fabs(v9[k]));
    if (sc == 0.0) sc = 1.0;
    for (int k = 0; k < 9; ++k) {
        W3[k] = dd(v9[k], sc);
        U3[k] = V3[k] = (k % 4 == 0) ? 1.0 : 0.0;
    }
    if (svd_core(3, W3, 3, U3, V3, sc, s3) < 0) status = ES_STATUS_SVD;
    s3[2] = 0.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            E[r * 3 + c] = da(da(dm(dm(U3[r * 3], s3[0]), V3[c * 3]), dm(dm(U3[r * 3 + 1], s3[1]), V3[c * 3 + 1])),
                              dm(dm(U3[r * 3 + 2], s3[2]), V3[c * 3 + 2]));
    return status;
}

/* compute_E_21_nonminimal over the m >= 8 pairs idx[0..m-1]; S is m x 9 scratch.  Returns 0, or ES_STATUS_SVD. */
ES_BIG int es_nonminimal(const double* b1, const double* b2, const int32_t* idx, int m, double* S, double* E) {
    double scale = 0.0;
    for (int i = 0; i < m; ++i) {
        const double* x1 = b1 + 3 * (size_t)idx[i];
        const double* x2 = b2 + 3 * (size_t)idx[i];
        for (int a = 0; a < 3; ++a)
            for (int c = 0; c < 3; ++c) {
                const double v = dm(x2[a], x1[c]);
                S[(size_t)i * 9 + 3 * a + c] = v;
                scale = es_max(scale, fabs(v));
            }
    }
    if (scale == 0.0) scale = 1.0;
    double v9[9];
    int status = es_svd_n9(m, S, scale, v9, NULL, NULL);
    status |= es_rank2(v9, E);
    return status;
}
