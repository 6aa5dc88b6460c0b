/* pnp_oracle.c -- CPU restatement of solve::pnp_solver (src/stella_vslam/solve/pnp_solver.cc) in the evaluation order of the
 * device code (stella_vslam_b200/csrc/epnp.cuh): sums left to right in index order, no contraction (-ffp-contract=off), float
 * exactly where the reference stores float.  The pieces of Eigen it uses are restated from Eigen 3.3/3.4's algorithms:
 *   JacobiSVD (two-sided, cyclic sweeps, threshold max(DBL_MIN, 2 eps maxDiag), sign flip of U, descending sort), square or
 *   preconditioned by ColPivHouseholderQR when rows > cols; rank() and solve(); HouseholderQR::solve.
 * Eigen's vectorised reductions are not reproduced: every sum runs left to right.  Test infrastructure, compiled on first use. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#define MAX_SWEEPS 64

static inline double dm(double a, double b) { return a * b; }
static inline double da(double a, double b) { return a + b; }
static inline double ds(double a, double b) { return a - b; }
static inline double dd(double a, double b) { return a / b; }
static inline double dot3(const double* a, const double* b) { return da(da(dm(a[0], b[0]), dm(a[1], b[1])), dm(a[2], b[2])); }

/* apply_rotation_in_the_plane(x, y, (c, s)) on one element pair */
static inline void rot2(double* x, double* y, double c, double s) {
    const double xi = *x, yi = *y;
    *x = da(dm(c, xi), dm(s, yi));
    *y = da(dm(-s, xi), dm(c, yi));
}

/* real_2x2_jacobi_svd on (m00 m01; m10 m11): j_left = (cl, sl), j_right = (cr, sr) */
static void jacobi_2x2(double m00, double m01, double m10, double m11, double* cl, double* sl, double* cr, double* sr) {
    double c1 = 1.0, s1 = 0.0;
    const double t = da(m00, m11), d = ds(m10, m01);
    if (!(fabs(d) < DBL_MIN)) {
        const double u = dd(t, d);
        const double tmp = sqrt(da(1.0, dm(u, u)));
        s1 = dd(1.0, tmp);
        c1 = dd(u, tmp);
    }
    if (!(c1 == 1.0 && s1 == 0.0)) {
        rot2(&m00, &m10, c1, s1);
        rot2(&m01, &m11, c1, s1);
    }
    double c = 1.0, s = 0.0;
    const double deno = dm(2.0, fabs(m01));
    if (!(deno < DBL_MIN)) {
        const double tau = dd(ds(m00, m11), deno);
        const double w = sqrt(da(dm(tau, tau), 1.0));
        const double tt = tau > 0.0 ? dd(1.0, da(tau, w)) : dd(1.0, ds(tau, w));
        const double sign_t = tt > 0.0 ? 1.0 : -1.0;
        const double n = dd(1.0, sqrt(da(dm(tt, tt), 1.0)));
        s = dm(dm(dm(-sign_t, dd(m01, fabs(m01))), fabs(tt)), n);
        c = n;
    }
    *cr = c;
    *sr = s;
    *cl = ds(dm(c1, c), dm(s1, -s));
    *sl = da(dm(c1, -s), dm(s1, c));
}

/* Sweeps of JacobiSVD on the n x n row-major W; U has m rows (row-major, stride m, columns p, q rotated), V is n x n or NULL.
 * Then singular values (scaled back), sign flip of U's columns and the descending sort.  Returns the number of nonzero singular
 * values, or -1 when the sweeps did not converge. */
static int svd_core(int n, double* W, int m, double* U, double* V, double scale, double* sv) {
    double max_diag = 0.0;
    for (int i = 0; i < n; ++i)
        if (fabs(W[i * n + i]) > max_diag || i == 0) max_diag = fabs(W[i * n + i]);
    const double precision = 2.0 * DBL_EPSILON;
    int finished = 0, sweeps = 0;
    while (!finished) {
        if (sweeps == MAX_SWEEPS) return -1;
        ++sweeps;
        finished = 1;
        for (int p = 1; p < n; ++p)
            for (int q = 0; q < p; ++q) {
                const double pm = dm(precision, max_diag);
                const double threshold = DBL_MIN < pm ? pm : DBL_MIN;
                if (!(fabs(W[p * n + q]) > threshold || fabs(W[q * n + p]) > threshold)) continue;
                finished = 0;
                double cl, sl, cr, sr;
                jacobi_2x2(W[p * n + p], W[p * n + q], W[q * n + p], W[q * n + q], &cl, &sl, &cr, &sr);
                if (!(cl == 1.0 && sl == 0.0)) {
                    for (int k = 0; k < n; ++k) rot2(&W[p * n + k], &W[q * n + k], cl, sl);
                    for (int k = 0; k < m; ++k) rot2(&U[k * m + p], &U[k * m + q], cl, sl);
                }
                if (!(cr == 1.0 && -sr == 0.0)) {
                    for (int k = 0; k < n; ++k) rot2(&W[k * n + p], &W[k * n + q], cr, -sr);
                    if (V)
                        for (int k = 0; k < n; ++k) rot2(&V[k * n + p], &V[k * n + q], cr, -sr);
                }
                const double dp = fabs(W[p * n + p]), dq = fabs(W[q * n + q]);
                const double dmx = dp < dq ? dq : dp;
                if (max_diag < dmx) max_diag = dmx;
            }
    }
    for (int i = 0; i < n; ++i) {
        const double a = W[i * n + i];
        sv[i] = fabs(a);
        if (a < 0.0)
            for (int k = 0; k < m; ++k) U[k * m + i] = -U[k * m + i];
    }
    for (int i = 0; i < n; ++i) sv[i] = dm(sv[i], scale);
    int nonzero = n;
    for (int i = 0; i < n; ++i) {
        int pos = i;
        for (int k = i + 1; k < n; ++k)
            if (sv[k] > sv[pos]) pos = k;
        if (sv[pos] == 0.0) {
            nonzero = i;
            break;
        }
        if (pos != i) {
            double t = sv[i];
            sv[i] = sv[pos];
            sv[pos] = t;
            for (int k = 0; k < m; ++k) {
                t = U[k * m + i];
                U[k * m + i] = U[k * m + pos];
                U[k * m + pos] = t;
            }
            if (V)
                for (int k = 0; k < n; ++k) {
                    t = V[k * n + i];
                    V[k * n + i] = V[k * n + pos];
                    V[k * n + pos] = t;
                }
        }
    }
    return nonzero;
}

static double max_abs(const double* A, int count) {
    double s = 0.0;
    for (int k = 0; k < count; ++k)
        if (fabs(A[k]) > s) s = fabs(A[k]);
    return s == 0.0 ? 1.0 : s;
}

/* JacobiSVD of a square n x n (row-major A) with full U (and V when V != NULL).  W is n*n scratch.  Returns as svd_core. */
int orc_svd_square(int n, const double* A, double* W, double* U, double* V, double* sv) {
    const double scale = max_abs(A, n * n);
    for (int k = 0; k < n * n; ++k) {
        W[k] = dd(A[k], scale);
        U[k] = (k % (n + 1) == 0) ? 1.0 : 0.0;
        if (V) V[k] = U[k];
    }
    return svd_core(n, W, n, U, V, scale, sv);
}

/* makeHouseholderInPlace on v[0], v[stride], ... (len entries): the essential part overwrites v[1..], returns tau and beta */
static void make_householder(double* v, int len, int stride, double* tau, double* beta) {
    double tail = 0.0;
    for (int i = 1; i < len; ++i) tail = (i == 1) ? dm(v[i * stride], v[i * stride]) : da(tail, dm(v[i * stride], v[i * stride]));
    const double c0 = v[0];
    if (tail <= DBL_MIN) {
        *tau = 0.0;
        *beta = c0;
        for (int i = 1; i < len; ++i) v[i * stride] = 0.0;
        return;
    }
    double b = sqrt(da(dm(c0, c0), tail));
    if (c0 >= 0.0) b = -b;
    const double den = ds(c0, b);
    for (int i = 1; i < len; ++i) v[i * stride] = dd(v[i * stride], den);
    *tau = dd(ds(b, c0), b);
    *beta = b;
}

/* applyHouseholderOnTheLeft to the block B (rows x cols, row-major stride ldb) with essential ess[0..rows-2] (stride es) */
static void apply_householder_left(double* B, int rows, int cols, int ldb, const double* ess, int es, double tau) {
    if (rows == 1) {
        const double f = ds(1.0, tau);
        for (int j = 0; j < cols; ++j) B[j] = dm(B[j], f);
        return;
    }
    if (tau == 0.0) return;
    for (int j = 0; j < cols; ++j) {
        double tmp = dm(ess[0], B[ldb + j]);
        for (int i = 1; i < rows - 1; ++i) tmp = da(tmp, dm(ess[i * es], B[(1 + i) * ldb + j]));
        tmp = da(tmp, B[j]);
        B[j] = ds(B[j], dm(tau, tmp));
        for (int i = 0; i < rows - 1; ++i) B[(1 + i) * ldb + j] = ds(B[(1 + i) * ldb + j], dm(dm(tau, ess[i * es]), tmp));
    }
}

static double col_norm(const double* A, int ld, int r0, int r1, int j) {
    double s = 0.0;
    for (int i = r0; i < r1; ++i) s = (i == r0) ? dm(A[i * ld + j], A[i * ld + j]) : da(s, dm(A[i * ld + j], A[i * ld + j]));
    return sqrt(s);
}

/* JacobiSVD<MatX_t>(A 6 x k, ComputeFullU | ComputeFullV).solve(rhs) for k in {3, 4, 5}: ColPivHouseholderQR preconditioner, sweeps
 * on R, rank() and the solve over the singular values above the rank threshold.  Returns the rank, or -1 (no convergence). */
int orc_svd_solve_6xk(int k, const double* A, const double* rhs, double* x, double* sv_out) {
    double S[30], U[36], W[25], V[25], sv[5], htau[5], cn_upd[5], cn_dir[5];
    int perm[5];
    const double scale = max_abs(A, 6 * k);
    for (int t = 0; t < 6 * k; ++t) S[t] = dd(A[t], scale);
    for (int j = 0; j < k; ++j) {
        cn_dir[j] = col_norm(S, k, 0, 6, j);
        cn_upd[j] = cn_dir[j];
        perm[j] = j;
    }
    const double norm_downdate_threshold = sqrt(DBL_EPSILON);
    for (int c = 0; c < k; ++c) {
        int big = c;
        for (int j = c + 1; j < k; ++j)
            if (cn_upd[j] > cn_upd[big]) big = j;
        if (big != c) {
            for (int i = 0; i < 6; ++i) {
                const double t = S[i * k + c];
                S[i * k + c] = S[i * k + big];
                S[i * k + big] = t;
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
        make_householder(&S[c * k + c], 6 - c, k, &htau[c], &beta);
        S[c * k + c] = beta;
        if (k - c - 1 > 0) apply_householder_left(&S[c * k + c + 1], 6 - c, k - c - 1, k, &S[(c + 1) * k + c], k, htau[c]);
        for (int j = c + 1; j < k; ++j) {
            if (cn_upd[j] == 0.0) continue;
            double temp = dd(fabs(S[c * k + j]), cn_upd[j]);
            temp = dm(da(1.0, temp), ds(1.0, temp));
            temp = temp < 0.0 ? 0.0 : temp;
            const double r = dd(cn_upd[j], cn_dir[j]);
            const double temp2 = dm(temp, dm(r, r));
            if (temp2 <= norm_downdate_threshold) {
                cn_dir[j] = col_norm(S, k, c + 1, 6, j);
                cn_upd[j] = cn_dir[j];
            } else {
                cn_upd[j] = dm(cn_upd[j], sqrt(temp));
            }
        }
    }
    /* householderQ().evalTo(U): identity, then the reflectors from the last to the first on the bottom-right corners */
    for (int t = 0; t < 36; ++t) U[t] = (t % 7 == 0) ? 1.0 : 0.0;
    for (int c = k - 1; c >= 0; --c) apply_householder_left(&U[c * 6 + c], 6 - c, 6 - c, 6, &S[(c + 1) * k + c], k, htau[c]);
    for (int i = 0; i < k; ++i)
        for (int j = 0; j < k; ++j) {
            W[i * k + j] = j >= i ? S[i * k + j] : 0.0;
            V[i * k + j] = (i == perm[j]) ? 1.0 : 0.0;
        }
    const int nonzero = svd_core(k, W, 6, U, V, scale, sv);
    if (nonzero < 0) return -1;
    const double thr0 = dm(sv[0], dm((double)k, DBL_EPSILON));
    const double thr = thr0 > DBL_MIN ? thr0 : DBL_MIN;
    int i = nonzero - 1;
    while (i >= 0 && sv[i] < thr) --i;
    const int rank = i + 1;
    double tmp[5];
    for (int j = 0; j < rank; ++j) {
        double s = dm(U[j], rhs[0]);
        for (int r = 1; r < 6; ++r) s = da(s, dm(U[r * 6 + j], rhs[r]));
        tmp[j] = dm(dd(1.0, sv[j]), s);
    }
    for (int r = 0; r < k; ++r) {
        double s = 0.0;
        for (int j = 0; j < rank; ++j) s = (j == 0) ? dm(V[r * k + j], tmp[j]) : da(s, dm(V[r * k + j], tmp[j]));
        x[r] = s;
    }
    if (sv_out)
        for (int j = 0; j < k; ++j) sv_out[j] = sv[j];
    return rank;
}

/* A.householderQr().solve(b) for a 6 x 4 A (row-major) */
void orc_householder_qr_solve_6x4(const double* A_in, const double* b, double* x) {
    double A[24], c[6], tau[4];
    memcpy(A, A_in, sizeof A);
    memcpy(c, b, sizeof c);
    for (int k = 0; k < 4; ++k) {
        double beta;
        make_householder(&A[k * 4 + k], 6 - k, 4, &tau[k], &beta);
        A[k * 4 + k] = beta;
        if (4 - k - 1 > 0) apply_householder_left(&A[k * 4 + k + 1], 6 - k, 4 - k - 1, 4, &A[(k + 1) * 4 + k], 4, tau[k]);
    }
    for (int k = 0; k < 4; ++k) apply_householder_left(&c[k], 6 - k, 1, 1, &A[(k + 1) * 4 + k], 4, tau[k]);
    for (int i = 3; i >= 0; --i) {
        if (c[i] == 0.0) continue;
        c[i] = dd(c[i], A[i * 4 + i]);
        for (int j = 0; j < i; ++j) c[j] = ds(c[j], dm(c[i], A[j * 4 + i]));
    }
    for (int i = 0; i < 4; ++i) x[i] = c[i];
}

/* ---------------------------------------------------------------------------------------------------------------------------- */
/* EPnP (pnp_solver::compute_pose and helpers) over points i = idx ? idx[j] : j, j < n                                          */

typedef struct {
    const double* b;
    const double* p;
    const int32_t* idx;
    int n;
} pts_t;

static inline const double* PB(const pts_t* s, int j) { return s->b + 3 * (size_t)(s->idx ? s->idx[j] : j); }
static inline const double* PP(const pts_t* s, int j) { return s->p + 3 * (size_t)(s->idx ? s->idx[j] : j); }

typedef struct {
    double cws[4][3];
    double CC_inv[9];
} epnp_basis_t;

static void alpha_of(const epnp_basis_t* E, const double* p, double a[4]) {
    const double d[3] = {ds(p[0], E->cws[0][0]), ds(p[1], E->cws[0][1]), ds(p[2], E->cws[0][2])};
    for (int r = 0; r < 3; ++r) a[1 + r] = dot3(&E->CC_inv[3 * r], d);
    a[0] = ds(ds(ds(1.0, a[1]), a[2]), a[3]);
}

/* estimate_R_and_t with the pcs of compute_pcs built on the fly from the alphas and ccs */
static int estimate_R_and_t(const pts_t* s, const epnp_basis_t* E, const double ccs[4][3], double flip, double R[9], double t[3]) {
    const int n = s->n;
    double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j) {
        double a[4], pc[3];
        alpha_of(E, PP(s, j), a);
        for (int c = 0; c < 3; ++c) pc[c] = dm(da(da(da(dm(a[0], ccs[0][c]), dm(a[1], ccs[1][c])), dm(a[2], ccs[2][c])), dm(a[3], ccs[3][c])), flip);
        for (int c = 0; c < 3; ++c) {
            pc0[c] = da(pc0[c], pc[c]);
            pw0[c] = da(pw0[c], PP(s, j)[c]);
        }
    }
    for (int c = 0; c < 3; ++c) {
        pc0[c] = dd(pc0[c], (double)n);
        pw0[c] = dd(pw0[c], (double)n);
    }
    double CM[9] = {0};
    for (int j = 0; j < n; ++j) {
        double a[4], dc[3], dw[3];
        alpha_of(E, PP(s, j), a);
        for (int c = 0; c < 3; ++c) {
            dc[c] = ds(dm(da(da(da(dm(a[0], ccs[0][c]), dm(a[1], ccs[1][c])), dm(a[2], ccs[2][c])), dm(a[3], ccs[3][c])), flip), pc0[c]);
            dw[c] = ds(PP(s, j)[c], pw0[c]);
        }
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) CM[r * 3 + c] = da(CM[r * 3 + c], dm(dc[r], dw[c]));
    }
    double W[9], U[9], V[9], sv[3];
    if (orc_svd_square(3, CM, W, U, V, sv) < 0) return -1;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[r * 3 + c] = da(da(dm(U[r * 3], V[c * 3]), dm(U[r * 3 + 1], V[c * 3 + 1])), dm(U[r * 3 + 2], V[c * 3 + 2]));
    const double det = da(ds(dm(R[0], ds(dm(R[4], R[8]), dm(R[5], R[7]))), dm(R[3], ds(dm(R[1], R[8]), dm(R[2], R[7])))),
                          dm(R[6], ds(dm(R[1], R[5]), dm(R[2], R[4]))));
    if (det < 0) {
        const double SGM[9] = {1, 0, 0, 0, 1, 0, 0, 0, -1};
        double T[9];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                T[r * 3 + c] = da(da(dm(U[r * 3], SGM[c]), dm(U[r * 3 + 1], SGM[3 + c])), dm(U[r * 3 + 2], SGM[6 + c]));
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) R[r * 3 + c] = da(da(dm(T[r * 3], V[c * 3]), dm(T[r * 3 + 1], V[c * 3 + 1])), dm(T[r * 3 + 2], V[c * 3 + 2]));
    }
    for (int r = 0; r < 3; ++r) t[r] = ds(pc0[r], dot3(&R[r * 3], pw0));
    return 0;
}

static double reprojection_error(const pts_t* s, const double R[9], const double t[3]) {
    double sum = 0.0;
    for (int j = 0; j < s->n; ++j) {
        const double* pw = PP(s, j);
        const double pc[3] = {da(dot3(&R[0], pw), t[0]), da(dot3(&R[3], pw), t[1]), da(dot3(&R[6], pw), t[2])};
        const double cosang = dd(dot3(pc, PB(s, j)), sqrt(dot3(pc, pc)));
        sum = da(sum, ds(1.0, cosang));
    }
    return dd(sum, (double)s->n);
}

static void find_initial_betas(const double L[60], const double rho[6], int N, double betas[4], int* status) {
    static const int cols[3][5] = {{0, 1, 2, -1, -1}, {0, 1, 2, 3, 4}, {0, 1, 3, 6, -1}};
    const int k = N == 2 ? 3 : (N == 3 ? 5 : 4);
    double A[30], b[5] = {0, 0, 0, 0, 0}; /* defined values when the sweeps hit their bound (status -1) */
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < k; ++j) A[i * k + j] = L[i * 10 + cols[N - 2][j]];
    if (orc_svd_solve_6xk(k, A, rho, b, NULL) < 0) *status = -1;
    if (N == 4) {
        if (b[0] < 0) {
            betas[0] = sqrt(-b[0]);
            betas[1] = dd(-b[1], betas[0]);
            betas[2] = dd(-b[2], betas[0]);
            betas[3] = dd(-b[3], betas[0]);
        } else {
            betas[0] = sqrt(b[0]);
            betas[1] = dd(b[1], betas[0]);
            betas[2] = dd(b[2], betas[0]);
            betas[3] = dd(b[3], betas[0]);
        }
        return;
    }
    if (b[0] < 0) {
        betas[0] = sqrt(-b[0]);
        betas[1] = (b[2] < 0) ? sqrt(-b[2]) : 0.0;
    } else {
        betas[0] = sqrt(b[0]);
        betas[1] = (b[2] > 0) ? sqrt(b[2]) : 0.0;
    }
    if (b[1] < 0) betas[0] = -betas[0];
    betas[2] = N == 3 ? dd(b[3], betas[0]) : 0.0;
    betas[3] = 0.0;
}

static void gauss_newton(const double L[60], const double rho[6], double betas[4], unsigned num_iter) {
    for (unsigned it = 0; it < num_iter; ++it) {
        double A[24], B[6], x[4];
        const double* b = betas;
        for (int i = 0; i < 6; ++i) {
            const double* l = &L[i * 10];
            A[i * 4 + 0] = da(da(da(dm(dm(2.0, l[0]), b[0]), dm(l[1], b[1])), dm(l[3], b[2])), dm(l[6], b[3]));
            A[i * 4 + 1] = da(da(da(dm(l[1], b[0]), dm(dm(2.0, l[2]), b[1])), dm(l[4], b[2])), dm(l[7], b[3]));
            A[i * 4 + 2] = da(da(da(dm(l[3], b[0]), dm(l[4], b[1])), dm(dm(2.0, l[5]), b[2])), dm(l[8], b[3]));
            A[i * 4 + 3] = da(da(da(dm(l[6], b[0]), dm(l[7], b[1])), dm(l[8], b[2])), dm(dm(2.0, l[9]), b[3]));
            double q = dm(dm(l[0], b[0]), b[0]);
            q = da(q, dm(dm(l[1], b[0]), b[1]));
            q = da(q, dm(dm(l[2], b[1]), b[1]));
            q = da(q, dm(dm(l[3], b[0]), b[2]));
            q = da(q, dm(dm(l[4], b[1]), b[2]));
            q = da(q, dm(dm(l[5], b[2]), b[2]));
            q = da(q, dm(dm(l[6], b[0]), b[3]));
            q = da(q, dm(dm(l[7], b[1]), b[3]));
            q = da(q, dm(dm(l[8], b[2]), b[3]));
            q = da(q, dm(dm(l[9], b[3]), b[3]));
            B[i] = ds(rho[i], q);
        }
        orc_householder_qr_solve_6x4(A, B, x);
        for (int i = 0; i < 4; ++i) betas[i] = da(betas[i], x[i]);
    }
}

/* pnp_solver::compute_pose.  R, t are written only when a candidate N has reproj_error < the running minimum (starting at DBL_MAX);
 * *wrote tells whether they were.  Returns the minimum (DBL_MAX when nothing was written), status -1 when an SVD did not converge. */
static double compute_pose(const pts_t* s, unsigned num_iter, double R[9], double t[3], int* wrote, int* status) {
    const int n = s->n;
    epnp_basis_t E;
    *wrote = 0;
    *status = 0;
    /* choose_control_points */
    double c0[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j)
        for (int c = 0; c < 3; ++c) c0[c] = da(c0[c], PP(s, j)[c]);
    for (int c = 0; c < 3; ++c) c0[c] = dd(c0[c], (double)n);
    double P[9] = {0};
    for (int j = 0; j < n; ++j) {
        double d[3];
        for (int c = 0; c < 3; ++c) d[c] = ds(PP(s, j)[c], c0[c]);
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) P[a * 3 + b] = da(P[a * 3 + b], dm(d[a], d[b]));
    }
    double W3[9], U3[9], V3[9], D[3];
    if (orc_svd_square(3, P, W3, U3, V3, D) < 0) *status = -1;
    for (int c = 0; c < 3; ++c) E.cws[0][c] = c0[c];
    for (int i = 1; i < 4; ++i) {
        const double k = sqrt(dd(D[i - 1], (double)n));
        for (int c = 0; c < 3; ++c) E.cws[i][c] = da(c0[c], dm(k, U3[c * 3 + i - 1]));
    }
    /* compute_barycentric_coordinates: CC_inv = V S U^T */
    double CC[9];
    for (int i = 0; i < 3; ++i)
        for (int r = 0; r < 3; ++r) CC[r * 3 + i] = ds(E.cws[i + 1][r], E.cws[0][r]);
    if (orc_svd_square(3, CC, W3, U3, V3, D) < 0) *status = -1;
    double S[9] = {0}, VS[9];
    for (int i = 0; i < 3; ++i) S[i * 4] = D[i] > 1e-6 ? dd(1.0, D[i]) : 0.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) VS[r * 3 + c] = da(da(dm(V3[r * 3], S[c]), dm(V3[r * 3 + 1], S[3 + c])), dm(V3[r * 3 + 2], S[6 + c]));
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            E.CC_inv[r * 3 + c] = da(da(dm(VS[r * 3], U3[c * 3]), dm(VS[r * 3 + 1], U3[c * 3 + 1])), dm(VS[r * 3 + 2], U3[c * 3 + 2]));
    /* M^T M over the 2n rows of compute_M, row by row */
    double MtM[144], W[144], U[144], sv[12];
    memset(MtM, 0, sizeof MtM);
    for (int j = 0; j < n; ++j) {
        double a[4], r1[12], r2[12];
        alpha_of(&E, PP(s, j), a);
        const double* b = PB(s, j);
        const double u = dd(b[0], b[2]), v = dd(b[1], b[2]);
        for (int i = 0; i < 4; ++i) {
            r1[3 * i] = a[i];
            r1[3 * i + 1] = 0.0;
            r1[3 * i + 2] = dm(-a[i], u);
            r2[3 * i] = 0.0;
            r2[3 * i + 1] = a[i];
            r2[3 * i + 2] = dm(-a[i], v);
        }
        for (int x = 0; x < 12; ++x)
            for (int y = 0; y < 12; ++y) MtM[x * 12 + y] = da(MtM[x * 12 + y], dm(r1[x], r1[y]));
        for (int x = 0; x < 12; ++x)
            for (int y = 0; y < 12; ++y) MtM[x * 12 + y] = da(MtM[x * 12 + y], dm(r2[x], r2[y]));
    }
    if (orc_svd_square(12, MtM, W, U, NULL, sv) < 0) {
        *status = -1;
        return DBL_MAX;
    }
    /* compute_L_6x10 and compute_rho */
    double L[60], rho[6];
    {
        static const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
        double dv[4][6][3];
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 6; ++j)
                for (int c = 0; c < 3; ++c) dv[i][j][c] = ds(U[(3 * pa[j] + c) * 12 + 11 - i], U[(3 * pb[j] + c) * 12 + 11 - i]);
        for (int j = 0; j < 6; ++j) {
            double* l = &L[j * 10];
            l[0] = dot3(dv[0][j], dv[0][j]);
            l[1] = dm(2.0, dot3(dv[0][j], dv[1][j]));
            l[2] = dot3(dv[1][j], dv[1][j]);
            l[3] = dm(2.0, dot3(dv[0][j], dv[2][j]));
            l[4] = dm(2.0, dot3(dv[1][j], dv[2][j]));
            l[5] = dot3(dv[2][j], dv[2][j]);
            l[6] = dm(2.0, dot3(dv[0][j], dv[3][j]));
            l[7] = dm(2.0, dot3(dv[1][j], dv[3][j]));
            l[8] = dm(2.0, dot3(dv[2][j], dv[3][j]));
            l[9] = dot3(dv[3][j], dv[3][j]);
            double d[3];
            for (int c = 0; c < 3; ++c) d[c] = ds(E.cws[pa[j]][c], E.cws[pb[j]][c]);
            rho[j] = dot3(d, d);
        }
    }
    double reproj_min = DBL_MAX;
    const int bearing_z_sign = PB(s, 0)[2] > 0;
    for (int N = 2; N <= 4; ++N) {
        double betas[4], ccs[4][3], Rc[9], tc[3];
        find_initial_betas(L, rho, N, betas, status);
        gauss_newton(L, rho, betas, num_iter);
        for (int i = 0; i < 4; ++i)
            for (int c = 0; c < 3; ++c) {
                double v = 0.0;
                for (int j = 0; j < 4; ++j) v = da(v, dm(betas[j], U[(3 * i + c) * 12 + 11 - j]));
                ccs[i][c] = v;
            }
        /* compute_pcs: the sign of the first local point's z against the first bearing's */
        double a[4];
        alpha_of(&E, PP(s, 0), a);
        const double pc0z = da(da(da(dm(a[0], ccs[0][2]), dm(a[1], ccs[1][2])), dm(a[2], ccs[2][2])), dm(a[3], ccs[3][2]));
        const double flip = ((pc0z > 0) != bearing_z_sign) ? -1.0 : 1.0;
        if (estimate_R_and_t(s, &E, ccs, flip, Rc, tc) < 0) *status = -1;
        const double err = reprojection_error(s, Rc, tc);
        if (err < reproj_min) {
            reproj_min = err;
            memcpy(R, Rc, sizeof Rc);
            memcpy(t, tc, sizeof tc);
            *wrote = 1;
        }
    }
    return reproj_min;
}

/* ---------------------------------------------------------------------------------------------------------------------------- */

/* util::cos (util/trigonometric.h) */
static inline float poly_cos(float v) {
    const float v2 = v * v;
    return 0.99940307f + v2 * (-0.49558072f + 0.03679168f * v2);
}
static float util_cos(float v) {
    const float PI = 3.14159265358979f;
    const float PI_2 = PI / 2.0f, TWO_PI = 2.0f * PI, INV_TWO_PI = 1.0f / TWO_PI, THREE_PI_2 = 3.0f * PI_2;
    v = v - (float)(int)floorf(v * INV_TWO_PI) * TWO_PI;
    v = (0.0f < v) ? v : -v;
    if (v < PI_2) return poly_cos(v);
    if (v < PI) return -poly_cos(PI - v);
    if (v < THREE_PI_2) return -poly_cos(v - PI);
    return poly_cos(TWO_PI - v);
}

/* max_cos_errors_ of the constructor */
float orc_max_cos_error(float scale_factor) { return util_cos((float)((double)scale_factor * (1.0 * M_PI / 180.0))); }

static unsigned check_inliers(const pts_t* s, const float* max_cos, const double R[9], const double t[3], uint8_t* flags, double* cost) {
    unsigned num = 0;
    double c = 0.0;
    for (int j = 0; j < s->n; ++j) {
        const double* pw = PP(s, j);
        const double pc[3] = {da(dot3(&R[0], pw), t[0]), da(dot3(&R[3], pw), t[1]), da(dot3(&R[6], pw), t[2])};
        const double cosang = dd(dot3(pc, PB(s, j)), sqrt(dot3(pc, pc)));
        const int in = (double)max_cos[j] < cosang;
        if (in) {
            c = da(c, ds(1.0, cosang));
            ++num;
        } else {
            c = da(c, (double)(1.0f - max_cos[j]));
        }
        if (flags) flags[j] = (uint8_t)in;
    }
    *cost = c;
    return num;
}

/* pnp_solver::compute_pose on n points.  R, t: in / out (written only when *wrote).  Returns 0, or -1 when an SVD did not converge. */
int orc_epnp_compute_pose(int n, const double* bearings, const double* points, unsigned num_iter, double* R, double* t, int* wrote,
                          double* reproj_error) {
    const pts_t s = {bearings, points, NULL, n};
    int status;
    *reproj_error = compute_pose(&s, num_iter, R, t, wrote, &status);
    return status;
}

/* find_via_ransac on given minimal sets (max_num_iter x 4).  Out: valid, best_iter (-1 none), num_inliers, min_cost, R, t (written
 * only when valid), flags (n; untouched on the early return).  max_cos: n floats (orc_max_cos_error of each match's scale factor).
 * Returns 0, or -1 when an SVD did not converge. */
int orc_pnp_ransac(int n, const double* bearings, const double* points, const float* max_cos, unsigned min_num_inliers,
                   unsigned gauss_newton_num_iter, unsigned max_num_iter, int recompute, const int32_t* min_sets, int* valid, int* best_iter,
                   int* num_inliers, double* min_cost, double* R, double* t, uint8_t* flags) {
    *valid = 0;
    *best_iter = -1;
    *num_inliers = 0;
    *min_cost = DBL_MAX;
    if ((unsigned)n < 4 || (unsigned)n < min_num_inliers) return 0;
    const pts_t all = {bearings, points, NULL, n};
    int status = 0;
    double best_R[9], best_t[3];
    for (unsigned it = 0; it < max_num_iter; ++it) {
        const pts_t ms = {bearings, points, min_sets + 4 * (size_t)it, 4};
        double Rh[9], th[3];
        int wrote, st;
        compute_pose(&ms, gauss_newton_num_iter, Rh, th, &wrote, &st);
        if (st) status = -1;
        /* a hypothesis whose compute_pose wrote nothing scores the previous hypothesis' pose again in the reference; that repeats
         * a cost which can never be strictly smaller, so it is rejected here (hypothesis 0: uninitialised in the reference) */
        if (!wrote) continue;
        double cost;
        const unsigned ni = check_inliers(&all, max_cos, Rh, th, NULL, &cost);
        if (ni > min_num_inliers && *min_cost > cost) {
            *min_cost = cost;
            *best_iter = (int)it;
            *num_inliers = (int)ni;
            memcpy(best_R, Rh, sizeof Rh);
            memcpy(best_t, th, sizeof th);
        }
    }
    *valid = *min_cost < DBL_MAX;
    if (!*valid) {
        memset(flags, 0, (size_t)n);
        return status;
    }
    double cost;
    check_inliers(&all, max_cos, best_R, best_t, flags, &cost);
    if (recompute) {
        int32_t idx_buf_n = 0;
        for (int j = 0; j < n; ++j) idx_buf_n += flags[j];
        int32_t* idx = (int32_t*)__builtin_alloca(sizeof(int32_t) * (size_t)(idx_buf_n > 0 ? idx_buf_n : 1));
        int m = 0;
        for (int j = 0; j < n; ++j)
            if (flags[j]) idx[m++] = j;
        const pts_t in = {bearings, points, idx, m};
        int wrote, st;
        compute_pose(&in, gauss_newton_num_iter, best_R, best_t, &wrote, &st);
        if (st) status = -1;
    }
    memcpy(R, best_R, sizeof best_R);
    memcpy(t, best_t, sizeof best_t);
    return status;
}
