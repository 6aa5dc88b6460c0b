/* pgo_oracle.c -- CPU restatement of optimize::graph_optimizer steps 4-5 (optimize/graph_optimizer.cc:254-302) for the tests.
 *
 * g2o::Sim3 (upstream tag 20230223_git), graph_opt_edge / shot_vertex, BaseFixedSizedEdge's central-difference Jacobian
 * (delta 1e-9), the 7x7 block Hessian, OptimizationAlgorithmLevenberg (tau 1e-5, rho rule, <= 10 trials) and terminate_action, in
 * the evaluation order of stella_vslam_b200/csrc/sim3.cuh, compiled without contraction.  The LM loop follows oracle/lba_oracle.c's
 * optimize_rounds.  The linear solve is a profile (envelope) Cholesky in the reverse Cuthill-McKee order the library uses, with
 * scalar rows instead of the library's 32x32 tiles: an exact SPD solve that agrees with the device's to rounding.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { double q[4], t[3], s; } sim3_t;

#define EPS 0.00001

static void quat_to_rot(const double* q, double* R) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
static void rot_to_quat(const double* R, double* q) {
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
        double qq[4];
        qq[i] = 0.5 * t;
        t = 0.5 / t;
        qq[3] = (R[k * 3 + j] - R[j * 3 + k]) * t;
        qq[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
        qq[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
        q[0] = qq[0]; q[1] = qq[1]; q[2] = qq[2]; q[3] = qq[3];
    }
}
static void quat_normalize(double* q) {
    if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
static void skew(const double* w, double* O) {
    O[0] = 0.0;   O[1] = -w[2]; O[2] = w[1];
    O[3] = w[2];  O[4] = 0.0;   O[5] = -w[0];
    O[6] = -w[1]; O[7] = w[0];  O[8] = 0.0;
}
static void mat3_mul(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
static void mat3_vec(const double* A, const double* v, double* out) {
    for (int i = 0; i < 3; ++i) out[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
static void cross(const double* a, const double* b, double* c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
static void quat_rotate(const double* q, const double* v, double* out) {
    double uv[3], c[3];
    cross(q, v, uv);
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    cross(q, uv, c);
    for (int i = 0; i < 3; ++i) out[i] = v[i] + q[3] * uv[i] + c[i];
}
static void quat_mul(const double* a, const double* b, double* r) {
    r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
}
static sim3_t s_mul(const sim3_t* a, const sim3_t* b) {
    sim3_t o;
    quat_mul(a->q, b->q, o.q);
    double rt[3];
    quat_rotate(a->q, b->t, rt);
    for (int i = 0; i < 3; ++i) o.t[i] = a->s * rt[i] + a->t[i];
    o.s = a->s * b->s;
    return o;
}
static sim3_t s_inverse(const sim3_t* a) {
    sim3_t o;
    const double qc[4] = {-a->q[0], -a->q[1], -a->q[2], a->q[3]};
    const double f = -1. / a->s;
    const double st[3] = {f * a->t[0], f * a->t[1], f * a->t[2]};
    quat_rotate(qc, st, o.t);
    memcpy(o.q, qc, sizeof(qc));
    o.s = 1. / a->s;
    quat_normalize(o.q);
    return o;
}
static void s_map(const sim3_t* a, const double* p, double* out) {
    double rp[3];
    quat_rotate(a->q, p, rp);
    for (int i = 0; i < 3; ++i) out[i] = a->s * rp[i] + a->t[i];
}
static sim3_t s_exp(const double* u) {
    const double omega[3] = {u[0], u[1], u[2]};
    const double ups[3] = {u[3], u[4], u[5]};
    const double sigma = u[6];
    const double theta = sqrt(omega[0] * omega[0] + omega[1] * omega[1] + omega[2] * omega[2]);
    double O[9], O2[9], R[9];
    skew(omega, O);
    sim3_t o;
    o.s = exp(sigma);
    mat3_mul(O, O, O2);
    double A, B, Cc;
    if (fabs(sigma) < EPS) {
        Cc = 1;
        if (theta < EPS) {
            A = 1. / 2.;
            B = 1. / 6.;
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + O[k] + O2[k];
        } else {
            const double theta2 = theta * theta;
            A = (1 - cos(theta)) / (theta2);
            B = (theta - sin(theta)) / (theta2 * theta);
            const double f1 = sin(theta) / theta, f2 = (1 - cos(theta)) / (theta * theta);
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + f1 * O[k] + f2 * O2[k];
        }
    } else {
        Cc = (o.s - 1) / sigma;
        if (theta < EPS) {
            const double sigma2 = sigma * sigma;
            A = ((sigma - 1) * o.s + 1) / sigma2;
            B = ((0.5 * sigma2 - sigma + 1) * o.s - 1) / (sigma2 * sigma);
            for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? 1.0 : 0.0) + O[k] + O2[k];
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
    rot_to_quat(R, o.q);
    double W[9];
    for (int k = 0; k < 9; ++k) W[k] = A * O[k] + B * O2[k] + ((k % 4 == 0) ? Cc : 0.0);
    mat3_vec(W, ups, o.t);
    return o;
}
static void lu3_solve(const double* Win, const double* rhs, double* x) {
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
static void s_log(const sim3_t* g, double* res) {
    const double sigma = log(g->s);
    double R[9], omega[3], O[9], O2[9];
    quat_to_rot(g->q, R);
    const double d = 0.5 * (R[0] + R[4] + R[8] - 1);
    const double dR[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    double A, B, Cc;
    if (fabs(sigma) < EPS) {
        Cc = 1;
        if (d > 1 - EPS) {
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
        Cc = (g->s - 1) / sigma;
        if (d > 1 - EPS) {
            const double sigma2 = sigma * sigma;
            for (int i = 0; i < 3; ++i) omega[i] = 0.5 * dR[i];
            A = ((sigma - 1) * g->s + 1) / (sigma2);
            B = ((0.5 * sigma2 - sigma + 1) * g->s - 1) / (sigma2 * sigma);
        } else {
            const double theta = acos(d);
            const double f = theta / (2 * sqrt(1 - d * d));
            for (int i = 0; i < 3; ++i) omega[i] = f * dR[i];
            const double theta2 = theta * theta;
            const double a = g->s * sin(theta);
            const double b = g->s * cos(theta);
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
    lu3_solve(W, g->t, ups);
    res[0] = omega[0]; res[1] = omega[1]; res[2] = omega[2];
    res[3] = ups[0]; res[4] = ups[1]; res[5] = ups[2];
    res[6] = sigma;
}
static sim3_t s_oplus(const sim3_t* est, const double* upd, int fix_scale) {
    const double u[7] = {upd[0], upd[1], upd[2], upd[3], upd[4], upd[5], fix_scale ? 0.0 : upd[6]};
    const sim3_t e = s_exp(u);
    return s_mul(&e, est);
}
static void edge_error(const sim3_t* m, const sim3_t* v1, const sim3_t* v2, double* e) {
    const sim3_t c1 = s_mul(m, v1);
    const sim3_t iv2 = s_inverse(v2);
    const sim3_t r = s_mul(&c1, &iv2);
    s_log(&r, e);
}
/* BaseFixedSizedEdge::linearizeOplus for one vertex side: J (7x7 row-major, rows = error components) */
static void edge_jacobian(const sim3_t* m, const sim3_t* v1, const sim3_t* v2, int side, int fix_scale, double* J) {
    const double delta = 1e-9, scalar = 1 / (2 * delta);
    for (int d = 0; d < 7; ++d) {
        double add[7] = {0, 0, 0, 0, 0, 0, 0}, ep[7], em[7];
        add[d] = delta;
        sim3_t p = s_oplus(side == 0 ? v1 : v2, add, fix_scale);
        if (side == 0) edge_error(m, &p, v2, ep); else edge_error(m, v1, &p, ep);
        add[d] = -delta;
        p = s_oplus(side == 0 ? v1 : v2, add, fix_scale);
        if (side == 0) edge_error(m, &p, v2, em); else edge_error(m, v1, &p, em);
        for (int k = 0; k < 7; ++k) J[7 * k + d] = scalar * (ep[k] - em[k]);
    }
}

/* ---------------- exported Sim3 algebra (sim3_t = 8 doubles: q xyzw, t, s) ---------------- */
void orc_sim3_exp(const double* u, double* out) { sim3_t o = s_exp(u); memcpy(out, &o, sizeof(o)); }
void orc_sim3_log(const double* g, double* out) { s_log((const sim3_t*)g, out); }
void orc_sim3_mul(const double* a, const double* b, double* out) { sim3_t o = s_mul((const sim3_t*)a, (const sim3_t*)b); memcpy(out, &o, sizeof(o)); }
void orc_sim3_inverse(const double* a, double* out) { sim3_t o = s_inverse((const sim3_t*)a); memcpy(out, &o, sizeof(o)); }
void orc_sim3_map(const double* a, const double* p, double* out) { s_map((const sim3_t*)a, p, out); }
void orc_sim3_from_rts(const double* R, const double* t, double s, double* out) {
    sim3_t o;
    rot_to_quat(R, o.q);
    quat_normalize(o.q);
    memcpy(o.t, t, sizeof(o.t));
    o.s = s;
    memcpy(out, &o, sizeof(o));
}
void orc_edge_error(const double* m, const double* v1, const double* v2, double* e) {
    edge_error((const sim3_t*)m, (const sim3_t*)v1, (const sim3_t*)v2, e);
}
void orc_edge_jacobian(const double* m, const double* v1, const double* v2, int side, int fix_scale, double* J) {
    edge_jacobian((const sim3_t*)m, (const sim3_t*)v1, (const sim3_t*)v2, side, fix_scale, J);
}

/* ---------------- ordering and envelope ---------------- */
typedef struct { int* ptr; int* idx; } adj_t;
static int* g_deg;
static int by_deg(const void* a, const void* b) {
    const int x = *(const int*)a, y = *(const int*)b;
    if (g_deg[x] != g_deg[y]) return g_deg[x] < g_deg[y] ? -1 : 1;
    return x < y ? -1 : (x > y);
}
static int cmp_int(const void* a, const void* b) { const int x = *(const int*)a, y = *(const int*)b; return x < y ? -1 : (x > y); }

/* free-vertex adjacency (unique, sorted) */
static void build_adj(int nv, const uint8_t* fixed, int ne, const int32_t* e1, const int32_t* e2, adj_t* A) {
    int* cnt = (int*)calloc(nv + 1, sizeof(int));
    for (int e = 0; e < ne; ++e)
        if (!fixed[e1[e]] && !fixed[e2[e]]) { cnt[e1[e] + 1]++; cnt[e2[e] + 1]++; }
    for (int v = 0; v < nv; ++v) cnt[v + 1] += cnt[v];
    int* idx = (int*)malloc(sizeof(int) * (cnt[nv] + 1));
    int* fill = (int*)malloc(sizeof(int) * (nv + 1));
    memcpy(fill, cnt, sizeof(int) * nv);
    for (int e = 0; e < ne; ++e)
        if (!fixed[e1[e]] && !fixed[e2[e]]) { idx[fill[e1[e]]++] = e2[e]; idx[fill[e2[e]]++] = e1[e]; }
    int* ptr = (int*)calloc(nv + 1, sizeof(int));
    int w = 0;
    for (int v = 0; v < nv; ++v) {
        const int b = cnt[v], n = cnt[v + 1] - b;
        qsort(idx + b, n, sizeof(int), cmp_int);
        ptr[v] = w;
        for (int i = 0; i < n; ++i)
            if (i == 0 || idx[b + i] != idx[b + i - 1]) idx[w++] = idx[b + i];
    }
    ptr[nv] = w;
    free(cnt); free(fill);
    A->ptr = ptr; A->idx = idx;
}

/* reverse Cuthill-McKee: least-degree unvisited start (ties: index), BFS with neighbours by (degree, index), reversed */
int orc_rcm(int nv, const uint8_t* fixed, int ne, const int32_t* e1, const int32_t* e2, int32_t* order, int32_t* pos, int64_t* env_tiles) {
    adj_t A;
    build_adj(nv, fixed, ne, e1, e2, &A);
    int* deg = (int*)malloc(sizeof(int) * nv);
    for (int v = 0; v < nv; ++v) deg[v] = A.ptr[v + 1] - A.ptr[v];
    g_deg = deg;
    int* byd = (int*)malloc(sizeof(int) * nv);
    int nf = 0;
    for (int v = 0; v < nv; ++v) if (!fixed[v]) byd[nf++] = v;
    qsort(byd, nf, sizeof(int), by_deg);
    char* seen = (char*)calloc(nv, 1);
    int* ord = (int*)malloc(sizeof(int) * (nf + 1));
    int* nb = (int*)malloc(sizeof(int) * (nv + 1));
    int no = 0;
    for (int s = 0; s < nf; ++s) {
        const int st = byd[s];
        if (seen[st]) continue;
        seen[st] = 1;
        int head = no;
        ord[no++] = st;
        while (head < no) {
            const int u = ord[head++];
            int m = 0;
            for (int i = A.ptr[u]; i < A.ptr[u + 1]; ++i) if (!seen[A.idx[i]]) nb[m++] = A.idx[i];
            qsort(nb, m, sizeof(int), by_deg);
            for (int i = 0; i < m; ++i) { seen[nb[i]] = 1; ord[no++] = nb[i]; }
        }
    }
    for (int i = 0; i < nv; ++i) pos[i] = -1;
    for (int i = 0; i < nf; ++i) { order[i] = ord[nf - 1 - i]; pos[order[i]] = i; }
    if (env_tiles) { /* the library's 32x32-tile envelope, in doubles */
        const int n = 7 * nf, nt = (n + 31) / 32;
        int* ft = (int*)malloc(sizeof(int) * (nt + 1));
        for (int t = 0; t < nt; ++t) ft[t] = t;
        for (int p = 0; p < nf; ++p) {
            int fp = p;
            const int v = order[p];
            for (int i = A.ptr[v]; i < A.ptr[v + 1]; ++i) if (pos[A.idx[i]] < fp) fp = pos[A.idx[i]];
            for (int r = 7 * p; r < 7 * p + 7; ++r) if ((7 * fp) / 32 < ft[r / 32]) ft[r / 32] = (7 * fp) / 32;
        }
        int64_t env = 0;
        for (int t = 0; t < nt; ++t) env += (int64_t)(t - ft[t] + 1) * 1024;
        *env_tiles = env;
        free(ft);
    }
    free(A.ptr); free(A.idx); free(deg); free(byd); free(seen); free(ord); free(nb);
    return nf;
}

/* ---------------- the solve ---------------- */
typedef struct {
    int nv, ne, nf, n, fix_scale;
    const sim3_t* meas;
    const int32_t *e1, *e2;
    sim3_t* est;
    int32_t *order, *pos;
    int* first;            /* per scalar row: first column of the profile */
    int64_t* rowoff;       /* per scalar row: offset of L(r, first[r]) */
    double *L, *J, *err, *H, *b, *x;
} pgo_t;

static double chi2_of(pgo_t* S, const sim3_t* est) {
    double chi = 0, e[7];
    for (int k = 0; k < S->ne; ++k) {
        edge_error(&S->meas[k], &est[S->e1[k]], &est[S->e2[k]], e);
        double c = 0;
        for (int j = 0; j < 7; ++j) c += e[j] * e[j];
        chi += c;
    }
    return chi;
}

/* dense 7x7 blocks per (row pos, col pos) of the lower triangle in a scalar profile; H holds A (lower) before factorisation */
static double* prof(pgo_t* S, int r, int c) { return &S->H[S->rowoff[r] + (c - S->first[r])]; }

static void build_system(pgo_t* S) {
    memset(S->H, 0, sizeof(double) * S->rowoff[S->n]);
    memset(S->b, 0, sizeof(double) * S->n);
    double e[7];
    for (int k = 0; k < S->ne; ++k) {
        const int v[2] = {S->e1[k], S->e2[k]};
        const int p[2] = {S->pos[v[0]], S->pos[v[1]]};
        edge_error(&S->meas[k], &S->est[v[0]], &S->est[v[1]], e);
        double* Jk[2] = {S->J, S->J + 49};
        for (int s = 0; s < 2; ++s)
            if (p[s] >= 0) edge_jacobian(&S->meas[k], &S->est[v[0]], &S->est[v[1]], s, S->fix_scale, Jk[s]);
        for (int s = 0; s < 2; ++s) {
            if (p[s] < 0) continue;
            for (int a = 0; a < 7; ++a) {
                for (int c = 0; c <= a; ++c) {
                    double acc = 0;
                    for (int j = 0; j < 7; ++j) acc += Jk[s][7 * j + a] * Jk[s][7 * j + c];
                    *prof(S, 7 * p[s] + a, 7 * p[s] + c) += acc;
                }
                double acc = 0;
                for (int j = 0; j < 7; ++j) acc += Jk[s][7 * j + a] * (-e[j]);
                S->b[7 * p[s] + a] += acc;
            }
        }
        if (p[0] >= 0 && p[1] >= 0) {
            const int sr = p[0] > p[1] ? 0 : 1, sc = 1 - sr;
            for (int a = 0; a < 7; ++a)
                for (int c = 0; c < 7; ++c) {
                    double acc = 0;
                    for (int j = 0; j < 7; ++j) acc += Jk[sr][7 * j + a] * Jk[sc][7 * j + c];
                    *prof(S, 7 * p[sr] + a, 7 * p[sc] + c) += acc;
                }
        }
    }
}

/* profile Cholesky of H + lambda I and the two substitutions; 0 on a non-positive pivot */
static int solve_system(pgo_t* S, double lambda) {
    const int n = S->n;
    memcpy(S->L, S->H, sizeof(double) * S->rowoff[n]);
    for (int r = 0; r < n; ++r) S->L[S->rowoff[r] + (r - S->first[r])] += lambda;
    for (int r = 0; r < n; ++r) {
        const int fr = S->first[r];
        double* Lr = S->L + S->rowoff[r] - fr;
        for (int c = fr; c <= r; ++c) {
            const int fc = S->first[c];
            const double* Lc = S->L + S->rowoff[c] - fc;
            double v = Lr[c];
            for (int k = fr > fc ? fr : fc; k < c; ++k) v -= Lr[k] * Lc[k];
            if (c < r) {
                Lr[c] = v / Lc[c];
            } else {
                if (!(v > 0)) return 0;
                Lr[r] = sqrt(v);
            }
        }
    }
    for (int r = 0; r < n; ++r) {
        const double* Lr = S->L + S->rowoff[r] - S->first[r];
        double v = S->b[r];
        for (int k = S->first[r]; k < r; ++k) v -= Lr[k] * S->x[k];
        S->x[r] = v / Lr[r];
    }
    for (int r = n - 1; r >= 0; --r) {
        const double* Lr = S->L + S->rowoff[r] - S->first[r];
        S->x[r] /= Lr[r];
        for (int k = S->first[r]; k < r; ++k) S->x[k] -= Lr[k] * S->x[r];
    }
    return 1;
}

/* stats: [iterations, trials, chi2_init, chi2_final, lambda_init, lambda_final, envelope doubles (tiles), then the chi2 after every
 * iteration (max_iter entries)] */
int orc_graph_optimize(int nv, int ne, int fix_scale, const double* est_in, const uint8_t* fixed, const int32_t* e1, const int32_t* e2,
                       const double* meas, int np, const double* points, const int32_t* point_ref, int max_iter, double gain_thr,
                       double* est_out, double* pose_out, double* points_out, double* stats) {
    pgo_t S;
    memset(&S, 0, sizeof(S));
    S.nv = nv; S.ne = ne; S.fix_scale = fix_scale;
    S.meas = (const sim3_t*)meas; S.e1 = e1; S.e2 = e2;
    S.est = (sim3_t*)malloc(sizeof(sim3_t) * nv);
    memcpy(S.est, est_in, sizeof(sim3_t) * nv);
    S.order = (int32_t*)malloc(sizeof(int32_t) * (nv + 1));
    S.pos = (int32_t*)malloc(sizeof(int32_t) * nv);
    int64_t env_tiles = 0;
    S.nf = orc_rcm(nv, fixed, ne, e1, e2, S.order, S.pos, &env_tiles);
    S.n = 7 * S.nf;
    const int n = S.n;
    S.first = (int*)malloc(sizeof(int) * (n + 1));
    for (int p = 0; p < S.nf; ++p)
        for (int a = 0; a < 7; ++a) S.first[7 * p + a] = 7 * p;
    for (int k = 0; k < ne; ++k) {
        const int p1 = S.pos[e1[k]], p2 = S.pos[e2[k]];
        if (p1 < 0 || p2 < 0) continue;
        const int hi = p1 > p2 ? p1 : p2, lo = p1 > p2 ? p2 : p1;
        for (int a = 0; a < 7; ++a) if (7 * lo < S.first[7 * hi + a]) S.first[7 * hi + a] = 7 * lo;
    }
    S.rowoff = (int64_t*)malloc(sizeof(int64_t) * (n + 1));
    S.rowoff[0] = 0;
    for (int r = 0; r < n; ++r) S.rowoff[r + 1] = S.rowoff[r] + (r - S.first[r] + 1);
    S.H = (double*)malloc(sizeof(double) * (S.rowoff[n] + 1));
    S.L = (double*)malloc(sizeof(double) * (S.rowoff[n] + 1));
    S.J = (double*)malloc(sizeof(double) * 98);
    S.b = (double*)malloc(sizeof(double) * (n + 1));
    S.x = (double*)malloc(sizeof(double) * (n + 1));
    sim3_t* bk = (sim3_t*)malloc(sizeof(sim3_t) * nv);

    /* SparseOptimizer::optimize(max_iter) with OptimizationAlgorithmLevenberg and terminate_action */
    double lambda = 0, ni = 2, last_chi = 0, chi2_init = 0, lambda_init = 0, chi = 0;
    int it = 0, trials = 0, ok = 1, stop = 0;
    for (; it < max_iter && !stop && ok; ++it) {
        double current_chi = chi2_of(&S, S.est);
        build_system(&S);
        if (it == 0) { /* computeLambdaInit */
            double mx = 0;
            for (int r = 0; r < n; ++r) mx = fmax(mx, fabs(S.H[S.rowoff[r] + (r - S.first[r])]));
            lambda = 1e-5 * mx;
            lambda_init = lambda;
            chi2_init = current_chi;
            ni = 2;
        }
        double rho = 0;
        int qmax = 0;
        do {
            memcpy(bk, S.est, sizeof(sim3_t) * nv); /* push */
            const int ok2 = solve_system(&S, lambda);
            ++trials;
            if (ok2)
                for (int v = 0; v < nv; ++v)
                    if (S.pos[v] >= 0) S.est[v] = s_oplus(&bk[v], S.x + 7 * S.pos[v], fix_scale);
            double temp_chi = chi2_of(&S, S.est);
            if (!ok2) temp_chi = DBL_MAX;
            rho = current_chi - temp_chi;
            double scale = 0; /* computeScale */
            if (ok2) for (int j = 0; j < n; ++j) scale += S.x[j] * (lambda * S.x[j] + S.b[j]);
            scale = ok2 ? scale + 1e-3 : 1;
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
                memcpy(S.est, bk, sizeof(sim3_t) * nv); /* pop */
                if (!isfinite(lambda)) break;
            }
            qmax++;
        } while (rho < 0 && qmax < 10);
        if (qmax == 10 || rho == 0 || !isfinite(lambda)) ok = 0;
        chi = chi2_of(&S, S.est); /* terminate_action: computeActiveErrors, activeRobustChi2 */
        stats[8 + it] = chi;
        if (it == 0) {
            last_chi = chi;
        } else {
            const double gain = (last_chi - chi) / chi;
            last_chi = chi;
            if (gain >= 0 && gain < gain_thr) stop = 1;
        }
    }
    if (it == 0) chi2_init = chi = chi2_of(&S, S.est);

    /* write-back (:261-302) */
    memcpy(est_out, S.est, sizeof(sim3_t) * nv);
    for (int v = 0; v < nv; ++v) {
        double R[9];
        quat_to_rot(S.est[v].q, R);
        const float s = (float)S.est[v].s;
        double* P = pose_out + 16 * (size_t)v;
        for (int r = 0; r < 3; ++r) {
            P[4 * r] = R[3 * r]; P[4 * r + 1] = R[3 * r + 1]; P[4 * r + 2] = R[3 * r + 2];
            P[4 * r + 3] = S.est[v].t[r] / (double)s;
        }
        P[12] = 0; P[13] = 0; P[14] = 0; P[15] = 1;
    }
    if (points_out)
        for (int i = 0; i < np; ++i) {
            const int ref = point_ref[i];
            double pc[3];
            s_map((const sim3_t*)est_in + ref, points + 3 * (size_t)i, pc);
            const sim3_t inv = s_inverse(&S.est[ref]);
            s_map(&inv, pc, points_out + 3 * (size_t)i);
        }
    stats[0] = it; stats[1] = trials; stats[2] = chi2_init; stats[3] = chi; stats[4] = lambda_init; stats[5] = lambda;
    stats[6] = (double)env_tiles;
    free(S.est); free(S.order); free(S.pos); free(S.first); free(S.rowoff); free(S.H); free(S.L); free(S.J); free(S.b); free(S.x); free(bk);
    return 0;
}
