// epnp.cuh -- solve::pnp_solver (src/stella_vslam/solve/pnp_solver.cc) as device functions: EPnP (compute_pose and its helpers) and
// check_inliers, with the pieces of Eigen they use restated from Eigen 3.3/3.4's algorithms (Eigen is not a dependency):
//   JacobiSVD, square: scale by the max |entry|, cyclic two-sided sweeps (jacobi.cuh), sign flip of U's columns, descending sort;
//   JacobiSVD<MatX_t> of a 6 x k (k = 3, 4, 5): ColPivHouseholderQR preconditioner first (full U = Q, V = the column permutation),
//     then rank() = singular values >= max(s0 * k * eps, DBL_MIN) and solve() over those only;
//   HouseholderQR<6 x 4>::solve (gauss_newton).
// fp64 with explicit round-to-nearest intrinsics, sums left to right in index order: operation for operation the CPU restatement
// tests/pnp_oracle.c.  Eigen's vectorised reductions are not reproduced (DESIGN.md section 8).  One thread runs one problem; the
// 12 x 12 work matrices live in the thread's local memory (L1-resident).  The out-of-line functions have internal linkage, so more than
// one translation unit can include this header (essential_kernels.cu uses its SVD and Householder pieces).
#pragma once

#include "jacobi.cuh"

namespace b200 {
namespace pnp {

using tri::da;
using tri::dd;
using tri::dm;
using tri::ds;

__device__ __forceinline__ double dot3(const double* a, const double* b) { return da(da(dm(a[0], b[0]), dm(a[1], b[1])), dm(a[2], b[2])); }

// Sweeps of JacobiSVD on the n x n row-major W; U has m rows (row-major, stride m; columns p, q rotated), V is n x n or null.  Then
// the singular values (scaled back), the sign flip of U's columns and the descending sort.  Returns the number of nonzero singular
// values, or -1 when the sweeps did not converge.
static __device__ __noinline__ int svd_core(int n, double* W, int m, double* U, double* V, double scale, double* sv) {
    double max_diag = 0.0;
    for (int i = 0; i < n; ++i)
        if (fabs(W[i * n + i]) > max_diag || i == 0) max_diag = fabs(W[i * n + i]);
    const double precision = 2.0 * DBL_EPSILON;
    bool finished = false;
    int sweeps = 0;
    while (!finished) {
        if (sweeps == tri::kMaxSweeps) return -1;
        ++sweeps;
        finished = true;
        for (int p = 1; p < n; ++p)
            for (int q = 0; q < p; ++q) {
                const double pm = dm(precision, max_diag);
                const double threshold = DBL_MIN < pm ? pm : DBL_MIN;
                if (!(fabs(W[p * n + q]) > threshold || fabs(W[q * n + p]) > threshold)) continue;
                finished = false;
                double cl, sl, cr, sr;
                tri::jacobi_2x2(W[p * n + p], W[p * n + q], W[q * n + p], W[q * n + q], cl, sl, cr, sr);
                if (!(cl == 1.0 && sl == 0.0)) {
                    for (int k = 0; k < n; ++k) tri::rot2(W[p * n + k], W[q * n + k], cl, sl);
                    for (int k = 0; k < m; ++k) tri::rot2(U[k * m + p], U[k * m + q], cl, sl);
                }
                if (!(cr == 1.0 && -sr == 0.0)) {
                    for (int k = 0; k < n; ++k) tri::rot2(W[k * n + p], W[k * n + q], cr, -sr);
                    if (V)
                        for (int k = 0; k < n; ++k) tri::rot2(V[k * n + p], V[k * n + q], cr, -sr);
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

__device__ __forceinline__ double max_abs_or_one(const double* A, int count) {
    double s = 0.0;
    for (int k = 0; k < count; ++k)
        if (fabs(A[k]) > s) s = fabs(A[k]);
    return s == 0.0 ? 1.0 : s;
}

// JacobiSVD of a square n x n with full U (and V when non-null).  A is overwritten by the work matrix.
__device__ __forceinline__ int svd_square(int n, double* A, double* U, double* V, double* sv) {
    const double scale = max_abs_or_one(A, n * n);
    for (int k = 0; k < n * n; ++k) {
        A[k] = dd(A[k], scale);
        U[k] = (k % (n + 1) == 0) ? 1.0 : 0.0;
        if (V) V[k] = U[k];
    }
    return svd_core(n, A, n, U, V, scale, sv);
}

// makeHouseholderInPlace on v[0], v[stride], ... (len entries): the essential part overwrites v[1..]
__device__ __forceinline__ void make_householder(double* v, int len, int stride, double& tau, double& beta) {
    double tail = 0.0;
    for (int i = 1; i < len; ++i) tail = (i == 1) ? dm(v[i * stride], v[i * stride]) : da(tail, dm(v[i * stride], v[i * stride]));
    const double c0 = v[0];
    if (tail <= DBL_MIN) {
        tau = 0.0;
        beta = c0;
        for (int i = 1; i < len; ++i) v[i * stride] = 0.0;
        return;
    }
    double b = __dsqrt_rn(da(dm(c0, c0), tail));
    if (c0 >= 0.0) b = -b;
    const double den = ds(c0, b);
    for (int i = 1; i < len; ++i) v[i * stride] = dd(v[i * stride], den);
    tau = dd(ds(b, c0), b);
    beta = b;
}

// applyHouseholderOnTheLeft to the block B (rows x cols, row stride ldb) with the essential part ess[0..rows-2] (stride es)
__device__ __forceinline__ void apply_householder_left(double* B, int rows, int cols, int ldb, const double* ess, int es, double tau) {
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

__device__ __forceinline__ double col_norm(const double* A, int ld, int r0, int r1, int j) {
    double s = 0.0;
    for (int i = r0; i < r1; ++i) s = (i == r0) ? dm(A[i * ld + j], A[i * ld + j]) : da(s, dm(A[i * ld + j], A[i * ld + j]));
    return __dsqrt_rn(s);
}

// JacobiSVD<MatX_t>(A (6 x k row-major), ComputeFullU | ComputeFullV).solve(rhs).  Returns the rank, or -1 (no convergence).
static __device__ __noinline__ int svd_solve_6xk(int k, const double* A, const double* rhs, double* x) {
    double S[30], U[36], W[25], V[25], sv[5], htau[5], cn_upd[5], cn_dir[5];
    int perm[5];
    const double scale = max_abs_or_one(A, 6 * k);
    for (int t = 0; t < 6 * k; ++t) S[t] = dd(A[t], scale);
    for (int j = 0; j < k; ++j) {
        cn_dir[j] = col_norm(S, k, 0, 6, j);
        cn_upd[j] = cn_dir[j];
        perm[j] = j;
    }
    const double norm_downdate_threshold = __dsqrt_rn(DBL_EPSILON);
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
        make_householder(&S[c * k + c], 6 - c, k, htau[c], beta);
        S[c * k + c] = beta;
        if (k - c - 1 > 0) apply_householder_left(&S[c * k + c + 1], 6 - c, k - c - 1, k, &S[(c + 1) * k + c], k, htau[c]);
        for (int j = c + 1; j < k; ++j) {  // the norm downdate of LAPACK's xGEQPF, as ColPivHouseholderQR does it
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
                cn_upd[j] = dm(cn_upd[j], __dsqrt_rn(temp));
            }
        }
    }
    // householderQ().evalTo(U): identity, then the reflectors from the last to the first on the bottom-right corners
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
    return rank;
}

// A.householderQr().solve(b) for a 6 x 4 A (row-major; overwritten), b overwritten, x out
__device__ __forceinline__ void householder_qr_solve_6x4(double* A, double* c, double* x) {
    double tau[4];
    for (int k = 0; k < 4; ++k) {
        double beta;
        make_householder(&A[k * 4 + k], 6 - k, 4, tau[k], beta);
        A[k * 4 + k] = beta;
        if (4 - k - 1 > 0) apply_householder_left(&A[k * 4 + k + 1], 6 - k, 4 - k - 1, 4, &A[(k + 1) * 4 + k], 4, tau[k]);
    }
    for (int k = 0; k < 4; ++k) apply_householder_left(&c[k], 6 - k, 1, 1, &A[(k + 1) * 4 + k], 4, tau[k]);
    for (int i = 3; i >= 0; --i) {  // column-oriented back substitution, skipping a zero right-hand side as Eigen does
        if (c[i] == 0.0) continue;
        c[i] = dd(c[i], A[i * 4 + i]);
        for (int j = 0; j < i; ++j) c[j] = ds(c[j], dm(c[i], A[j * 4 + i]));
    }
    for (int i = 0; i < 4; ++i) x[i] = c[i];
}

// ---------------------------------------------------------------------------------------------------------------------------------
// EPnP over the points j < n of a problem, index idx ? idx[j] : j into its bearings / points (n x 3)

struct Pts {
    const double* b;
    const double* p;
    const int32_t* idx;
    int n;
    __device__ __forceinline__ const double* B(int j) const { return b + 3 * (size_t)(idx ? idx[j] : j); }
    __device__ __forceinline__ const double* P(int j) const { return p + 3 * (size_t)(idx ? idx[j] : j); }
};

struct Basis {
    double cws[4][3];
    double CC_inv[9];
};

__device__ __forceinline__ void alpha_of(const Basis& E, const double* p, double a[4]) {
    const double d[3] = {ds(p[0], E.cws[0][0]), ds(p[1], E.cws[0][1]), ds(p[2], E.cws[0][2])};
    for (int r = 0; r < 3; ++r) a[1 + r] = dot3(&E.CC_inv[3 * r], d);
    a[0] = ds(ds(ds(1.0, a[1]), a[2]), a[3]);
}

__device__ __forceinline__ double pcs_coord(const double a[4], const double ccs[4][3], int c) {
    return da(da(da(dm(a[0], ccs[0][c]), dm(a[1], ccs[1][c])), dm(a[2], ccs[2][c])), dm(a[3], ccs[3][c]));
}

// estimate_R_and_t, with compute_pcs' local points rebuilt on the fly from the alphas and ccs (flip = -1 inverts them)
static __device__ __noinline__ int estimate_R_and_t(const Pts& s, const Basis& E, const double (&ccs)[4][3], double flip, double* R, double* t) {
    const int n = s.n;
    double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j) {
        double a[4];
        alpha_of(E, s.P(j), a);
        for (int c = 0; c < 3; ++c) {
            pc0[c] = da(pc0[c], dm(pcs_coord(a, ccs, c), flip));
            pw0[c] = da(pw0[c], s.P(j)[c]);
        }
    }
    for (int c = 0; c < 3; ++c) {
        pc0[c] = dd(pc0[c], (double)n);
        pw0[c] = dd(pw0[c], (double)n);
    }
    double CM[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < n; ++j) {
        double a[4], dc[3], dw[3];
        alpha_of(E, s.P(j), a);
        for (int c = 0; c < 3; ++c) {
            dc[c] = ds(dm(pcs_coord(a, ccs, c), flip), pc0[c]);
            dw[c] = ds(s.P(j)[c], pw0[c]);
        }
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) CM[r * 3 + c] = da(CM[r * 3 + c], dm(dc[r], dw[c]));
    }
    double U[9], V[9], sv[3];
    if (svd_square(3, CM, U, V, sv) < 0) return -1;
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

// cos of the angle between R p + t and the bearing (check_inliers, reprojection_error)
__device__ __forceinline__ double cos_angle(const double* R, const double* t, const double* pw, const double* b) {
    const double pc[3] = {da(dot3(&R[0], pw), t[0]), da(dot3(&R[3], pw), t[1]), da(dot3(&R[6], pw), t[2])};
    return dd(dot3(pc, b), __dsqrt_rn(dot3(pc, pc)));
}

__device__ __forceinline__ double reprojection_error(const Pts& s, const double* R, const double* t) {
    double sum = 0.0;
    for (int j = 0; j < s.n; ++j) sum = da(sum, ds(1.0, cos_angle(R, t, s.P(j), s.B(j))));
    return dd(sum, (double)s.n);
}

__device__ __forceinline__ void find_initial_betas(const double* L, const double* rho, int N, double* betas, int& status) {
    const int k = N == 2 ? 3 : (N == 3 ? 5 : 4);
    double A[30], b[5] = {0, 0, 0, 0, 0};  // defined values when the sweeps hit their bound (status -1)
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < k; ++j) {
            const int col = N == 4 ? (j == 0 ? 0 : (j == 1 ? 1 : (j == 2 ? 3 : 6))) : j;  // L_6x4 takes columns 0, 1, 3, 6
            A[i * k + j] = L[i * 10 + col];
        }
    if (svd_solve_6xk(k, A, rho, b) < 0) status = -1;
    if (N == 4) {
        if (b[0] < 0) {
            betas[0] = __dsqrt_rn(-b[0]);
            betas[1] = dd(-b[1], betas[0]);
            betas[2] = dd(-b[2], betas[0]);
            betas[3] = dd(-b[3], betas[0]);
        } else {
            betas[0] = __dsqrt_rn(b[0]);
            betas[1] = dd(b[1], betas[0]);
            betas[2] = dd(b[2], betas[0]);
            betas[3] = dd(b[3], betas[0]);
        }
        return;
    }
    if (b[0] < 0) {
        betas[0] = __dsqrt_rn(-b[0]);
        betas[1] = (b[2] < 0) ? __dsqrt_rn(-b[2]) : 0.0;
    } else {
        betas[0] = __dsqrt_rn(b[0]);
        betas[1] = (b[2] > 0) ? __dsqrt_rn(b[2]) : 0.0;
    }
    if (b[1] < 0) betas[0] = -betas[0];
    betas[2] = N == 3 ? dd(b[3], betas[0]) : 0.0;
    betas[3] = 0.0;
}

static __device__ __noinline__ void gauss_newton(const double* L, const double* rho, double* betas, unsigned num_iter) {
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
        householder_qr_solve_6x4(A, B, x);
        for (int i = 0; i < 4; ++i) betas[i] = da(betas[i], x[i]);
    }
}

// pnp_solver::compute_pose.  R, t are written only when a candidate N has reproj_error < the running minimum (from DBL_MAX); `wrote`
// says whether they were.  Returns the minimum; status = -1 when an SVD did not converge.
static __device__ __noinline__ double compute_pose(const Pts& s, unsigned num_iter, double* R, double* t, bool& wrote, int& status) {
    const int n = s.n;
    Basis E;
    wrote = false;
    status = 0;
    // choose_control_points
    double c0[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j)
        for (int c = 0; c < 3; ++c) c0[c] = da(c0[c], s.P(j)[c]);
    for (int c = 0; c < 3; ++c) c0[c] = dd(c0[c], (double)n);
    double P[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < n; ++j) {
        double d[3];
        for (int c = 0; c < 3; ++c) d[c] = ds(s.P(j)[c], c0[c]);
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) P[a * 3 + b] = da(P[a * 3 + b], dm(d[a], d[b]));
    }
    double U3[9], V3[9], D[3];
    if (svd_square(3, P, U3, V3, D) < 0) status = -1;
    for (int c = 0; c < 3; ++c) E.cws[0][c] = c0[c];
    for (int i = 1; i < 4; ++i) {
        const double k = __dsqrt_rn(dd(D[i - 1], (double)n));
        for (int c = 0; c < 3; ++c) E.cws[i][c] = da(c0[c], dm(k, U3[c * 3 + i - 1]));
    }
    // compute_barycentric_coordinates: CC_inv = V S U^T with the pseudo-inverse of the singular values above 1e-6
    double CC[9];
    for (int i = 0; i < 3; ++i)
        for (int r = 0; r < 3; ++r) CC[r * 3 + i] = ds(E.cws[i + 1][r], E.cws[0][r]);
    if (svd_square(3, CC, U3, V3, D) < 0) status = -1;
    double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, VS[9];
    for (int i = 0; i < 3; ++i) S[i * 4] = D[i] > 1e-6 ? dd(1.0, D[i]) : 0.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) VS[r * 3 + c] = da(da(dm(V3[r * 3], S[c]), dm(V3[r * 3 + 1], S[3 + c])), dm(V3[r * 3 + 2], S[6 + c]));
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            E.CC_inv[r * 3 + c] = da(da(dm(VS[r * 3], U3[c * 3]), dm(VS[r * 3 + 1], U3[c * 3 + 1])), dm(VS[r * 3 + 2], U3[c * 3 + 2]));
    // M^T M over the 2n rows of compute_M, row by row
    // (the loops over W and U stay rolled: unrolled, the compiler would promote the 12 x 12 arrays to registers and spill them)
    double W[144], U[144], sv[12];
#pragma unroll 1
    for (int k = 0; k < 144; ++k) W[k] = 0.0;
    for (int j = 0; j < n; ++j) {
        double a[4], r1[12], r2[12];
        alpha_of(E, s.P(j), a);
        const double* b = s.B(j);
        const double u = dd(b[0], b[2]), v = dd(b[1], b[2]);
        for (int i = 0; i < 4; ++i) {
            r1[3 * i] = a[i];
            r1[3 * i + 1] = 0.0;
            r1[3 * i + 2] = dm(-a[i], u);
            r2[3 * i] = 0.0;
            r2[3 * i + 1] = a[i];
            r2[3 * i + 2] = dm(-a[i], v);
        }
#pragma unroll 1
        for (int x = 0; x < 12; ++x)
            for (int y = 0; y < 12; ++y) W[x * 12 + y] = da(W[x * 12 + y], dm(r1[x], r1[y]));
#pragma unroll 1
        for (int x = 0; x < 12; ++x)
            for (int y = 0; y < 12; ++y) W[x * 12 + y] = da(W[x * 12 + y], dm(r2[x], r2[y]));
    }
    if (svd_square(12, W, U, nullptr, sv) < 0) {
        status = -1;
        return DBL_MAX;
    }
    // compute_L_6x10 (U's columns 11 - i) and compute_rho
    double L[60], rho[6];
#pragma unroll 1
    for (int j = 0; j < 6; ++j) {
        const int pa = j < 3 ? 0 : (j < 5 ? 1 : 2), pb = j < 3 ? j + 1 : (j < 5 ? j - 1 : 3);
        double dv[4][3];
        for (int i = 0; i < 4; ++i)
            for (int c = 0; c < 3; ++c) dv[i][c] = ds(U[(3 * pa + c) * 12 + 11 - i], U[(3 * pb + c) * 12 + 11 - i]);
        double* l = &L[j * 10];
        l[0] = dot3(dv[0], dv[0]);
        l[1] = dm(2.0, dot3(dv[0], dv[1]));
        l[2] = dot3(dv[1], dv[1]);
        l[3] = dm(2.0, dot3(dv[0], dv[2]));
        l[4] = dm(2.0, dot3(dv[1], dv[2]));
        l[5] = dot3(dv[2], dv[2]);
        l[6] = dm(2.0, dot3(dv[0], dv[3]));
        l[7] = dm(2.0, dot3(dv[1], dv[3]));
        l[8] = dm(2.0, dot3(dv[2], dv[3]));
        l[9] = dot3(dv[3], dv[3]);
        double d[3];
        for (int c = 0; c < 3; ++c) d[c] = ds(E.cws[pa][c], E.cws[pb][c]);
        rho[j] = dot3(d, d);
    }
    double reproj_min = DBL_MAX;
    const bool bearing_z_sign = s.B(0)[2] > 0;
#pragma unroll 1
    for (int N = 2; N <= 4; ++N) {
        double betas[4], ccs[4][3], Rc[9], tc[3];
        find_initial_betas(L, rho, N, betas, status);
        gauss_newton(L, rho, betas, num_iter);
#pragma unroll 1
        for (int i = 0; i < 4; ++i)
            for (int c = 0; c < 3; ++c) {
                double v = 0.0;
                for (int j = 0; j < 4; ++j) v = da(v, dm(betas[j], U[(3 * i + c) * 12 + 11 - j]));
                ccs[i][c] = v;
            }
        // compute_pcs: the local points are inverted when the first one's z sign differs from the first bearing's
        double a[4];
        alpha_of(E, s.P(0), a);
        const double flip = ((pcs_coord(a, ccs, 2) > 0) != bearing_z_sign) ? -1.0 : 1.0;
        if (estimate_R_and_t(s, E, ccs, flip, Rc, tc) < 0) status = -1;
        const double err = reprojection_error(s, Rc, tc);
        if (err < reproj_min) {
            reproj_min = err;
            for (int k = 0; k < 9; ++k) R[k] = Rc[k];
            for (int k = 0; k < 3; ++k) t[k] = tc[k];
            wrote = true;
        }
    }
    return reproj_min;
}

}  // namespace pnp
}  // namespace b200
