/* transform_oracle.c -- CPU restatement of optimize::transform_optimizer::optimize (optimize/transform_optimizer.cc:20-158) for the
 * tests.  It reuses the g2o::Sim3 restatement of pgo_oracle.c (s_exp, s_mul, s_inverse, s_map, s_oplus, mat3_vec) by including that
 * file, so both oracles evaluate the algebra in the same order as stella_vslam_b200/csrc/sim3.cuh; compiled without contraction.
 */
#include "pgo_oracle.c"

/* One Sim3_12 vertex (transform_vertex: oplus = Sim3(update) * estimate, update[6] zeroed under fix_scale), a forward edge_12 and a
 * backward edge_21 per gathered pair (internal/sim3/forward_reproj_edge.h, backward_reproj_edge.h), Huber delta sqrt(chi_sq) in float,
 * the central-difference Jacobian above, OptimizationAlgorithmLevenberg without a terminate action, the round-1 outlier test, the
 * early return, optimize(num_iter) and the inlier count.  The outlier tests read the errors computed last: those of the last trial
 * state of the round.  The 7x7 damped system is solved by a dense Cholesky, as on the device.  Sums run over the pairs in order,
 * edge_12 before edge_21. */
typedef struct { int model; double fx, fy, cx, cy, cols, rows; } tcam_t;

static void t_cam(const double* c, tcam_t* o) {
    o->model = (int)c[0]; o->fx = c[1]; o->fy = c[2]; o->cx = c[3]; o->cy = c[4]; o->cols = c[5]; o->rows = c[6];
}
static void t_rigid(const double* R, const double* t, const double* p, double* out) {
    mat3_vec(R, p, out);
    for (int i = 0; i < 3; ++i) out[i] += t[i];
}
static void t_project(const tcam_t* c, const double* p, double* u) {
    const double pi = 3.14159265358979323846;
    if (c->model == 1) {
        const double theta = atan2(p[0], p[2]);
        const double phi = -asin(p[1] / sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
        u[0] = c->cols * (0.5 + theta / (2 * pi));
        u[1] = c->rows * (0.5 - phi / pi);
    } else {
        u[0] = c->fx * p[0] / p[2] + c->cx;
        u[1] = c->fy * p[1] / p[2] + c->cy;
    }
}
/* computeError at the camera-frame point pc mapped by S; returns chi2() = e . (w I e) */
static double t_edge(const sim3_t* S, const double* pc, const tcam_t* c, const float* obs, double w, double* e) {
    double p[3], u[2];
    s_map(S, pc, p);
    t_project(c, p, u);
    e[0] = (double)obs[0] - u[0];
    e[1] = (double)obs[1] - u[1];
    return e[0] * (w * e[0]) + e[1] * (w * e[1]);
}
/* side 0: edge_12 maps with Sim3_12; side 1: edge_21 maps with Sim3_12.inverse() */
static double t_edge_at(const sim3_t* S12, int side, const double* pc, const tcam_t* c, const float* obs, double w, double* e) {
    if (!side) return t_edge(S12, pc, c, obs, w, e);
    const sim3_t inv = s_inverse(S12);
    return t_edge(&inv, pc, c, obs, w, e);
}
static void t_jacobian(const sim3_t* S12, int side, const double* pc, const tcam_t* c, const float* obs, double w, int fix_scale, double* J) {
    const double delta = 1e-9, scalar = 1 / (2 * delta);
    for (int d = 0; d < 7; ++d) {
        double add[7] = {0, 0, 0, 0, 0, 0, 0}, ep[2], em[2];
        add[d] = delta;
        sim3_t p = s_oplus(S12, add, fix_scale);
        t_edge_at(&p, side, pc, c, obs, w, ep);
        add[d] = -delta;
        p = s_oplus(S12, add, fix_scale);
        t_edge_at(&p, side, pc, c, obs, w, em);
        J[d] = scalar * (ep[0] - em[0]);
        J[7 + d] = scalar * (ep[1] - em[1]);
    }
}
static double t_huber_weight(double e2, double delta) { return (e2 <= delta * delta) ? 1.0 : delta / sqrt(e2); }
static double t_huber_cost(double e2, double delta) { return (e2 <= delta * delta) ? e2 : 2 * sqrt(e2) * delta - delta * delta; }

typedef struct {
    int n, fix_scale;
    tcam_t c[2];
    const float *obs[2], *w[2];
    double* pc[2];      /* n x 3 camera-frame points: pc[0] = R_2w pos_w_2 + t_2w (edge_12), pc[1] = R_1w pos_w_1 + t_1w (edge_21) */
    uint8_t* keep;
    double delta;
} tprob_t;

/* robust chi2 of the active pairs at S, and with acc != NULL the 28 upper entries of H followed by b */
static double t_accumulate(const tprob_t* P, const sim3_t* S, double* acc) {
    double chi = 0;
    if (acc) memset(acc, 0, sizeof(double) * 35);
    for (int i = 0; i < P->n; ++i) {
        if (!P->keep[i]) continue;
        for (int side = 0; side < 2; ++side) {
            double e[2], J[14];
            const double w = (double)P->w[side][i];
            const double c2 = t_edge_at(S, side, P->pc[side] + 3 * i, &P->c[side], P->obs[side] + 2 * i, w, e);
            chi += t_huber_cost(c2, P->delta);
            if (!acc) continue;
            t_jacobian(S, side, P->pc[side] + 3 * i, &P->c[side], P->obs[side] + 2 * i, w, P->fix_scale, J);
            const double ww = w * t_huber_weight(c2, P->delta);
            int k = 0;
            for (int a = 0; a < 7; ++a)
                for (int b = a; b < 7; ++b) acc[k++] += ww * (J[a] * J[b] + J[7 + a] * J[7 + b]);
            for (int a = 0; a < 7; ++a) acc[28 + a] += -ww * (J[a] * e[0] + J[7 + a] * e[1]);
        }
    }
    return chi;
}
static int t_solve7(const double* Hu, const double* b, double lambda, double* x) {
    double A[49];
    int k = 0;
    for (int a = 0; a < 7; ++a)
        for (int c = a; c < 7; ++c) { A[a * 7 + c] = Hu[k]; A[c * 7 + a] = Hu[k]; ++k; }
    for (int a = 0; a < 7; ++a) { A[a * 8] += lambda; x[a] = b[a]; }
    for (int j = 0; j < 7; ++j) {
        double d = A[j * 7 + j];
        for (int kk = 0; kk < j; ++kk) d -= A[j * 7 + kk] * A[j * 7 + kk];
        if (!(d > 0) || !isfinite(d)) return 0;
        d = sqrt(d);
        A[j * 7 + j] = d;
        for (int i = j + 1; i < 7; ++i) {
            double sv = A[i * 7 + j];
            for (int kk = 0; kk < j; ++kk) sv -= A[i * 7 + kk] * A[j * 7 + kk];
            A[i * 7 + j] = sv / d;
        }
    }
    for (int i = 0; i < 7; ++i) {
        double sv = x[i];
        for (int kk = 0; kk < i; ++kk) sv -= A[i * 7 + kk] * x[kk];
        x[i] = sv / A[i * 8];
    }
    for (int i = 6; i >= 0; --i) {
        double sv = x[i];
        for (int kk = i + 1; kk < 7; ++kk) sv -= A[kk * 7 + i] * x[kk];
        x[i] = sv / A[i * 8];
    }
    return 1;
}
/* SparseOptimizer::optimize(iters): st[0] iterations, st[1] trials, st[2] chi2 of the state left, st[3] lambda_init, st[4] the
 * iteration whose LM step failed (-1: none).  *last is the state of the last trial (whose errors g2o holds afterwards). */
static void t_lm_round(const tprob_t* P, sim3_t* cur, sim3_t* last, int iters, double* st) {
    double acc[35], x[7], lambda = 0, ni = 2, cur_chi = 0;
    int it = 0, trials = 0, ok = 1;
    st[3] = 0;
    st[4] = -1;
    for (; P->n > 0 && it < iters && ok; ++it) {
        cur_chi = t_accumulate(P, cur, acc);
        if (it == 0) {
            double mx = 0;
            for (int a = 0, k = 0; a < 7; k += 7 - a, ++a) mx = fmax(mx, fabs(acc[k]));
            lambda = 1e-5 * mx;
            ni = 2;
            st[3] = lambda;
        }
        double rho = 0;
        int qmax = 0;
        do {
            const int ok2 = t_solve7(acc, acc + 28, lambda, x);
            ++trials;
            *last = ok2 ? s_oplus(cur, x, P->fix_scale) : *cur;
            double temp_chi = t_accumulate(P, last, NULL);
            if (!ok2) temp_chi = DBL_MAX;
            rho = cur_chi - temp_chi;
            double scale = 0;
            if (ok2) for (int j = 0; j < 7; ++j) scale += x[j] * (lambda * x[j] + acc[28 + j]);
            scale = ok2 ? scale + 1e-3 : 1;
            rho /= scale;
            if (rho > 0 && isfinite(temp_chi) && ok2) {
                double alpha = 1. - pow((2 * rho - 1), 3);
                alpha = fmin(alpha, 2. / 3.);
                lambda *= fmax(1. / 3., alpha);
                ni = 2;
                cur_chi = temp_chi;
                *cur = *last;
            } else {
                lambda *= ni;
                ni *= 2;
                if (!isfinite(lambda)) break;
            }
            qmax++;
        } while (rho < 0 && qmax < 10);
        if (qmax == 10 || rho == 0 || !isfinite(lambda)) { ok = 0; st[4] = it; }
    }
    st[0] = it;
    st[1] = trials;
    st[2] = it > 0 ? cur_chi : 0.0;
}

/* Exported edge pieces.  S12: Sim3_12 (8 doubles); pc: camera-frame point (3); cam: model, fx, fy, cx, cy, cols, rows. */
double orc_transform_edge(const double* S12, int side, const double* pc, const double* cam, const float* obs, float w, double* e) {
    tcam_t c;
    t_cam(cam, &c);
    return t_edge_at((const sim3_t*)S12, side, pc, &c, obs, (double)w, e);
}
void orc_transform_jacobian(const double* S12, int side, const double* pc, const double* cam, const float* obs, float w, int fix_scale, double* J) {
    tcam_t c;
    t_cam(cam, &c);
    t_jacobian((const sim3_t*)S12, side, pc, &c, obs, (double)w, fix_scale, J);
}

/* transform_optimizer(fix_scale, num_iter)::optimize on gathered pairs.  Returns num_inliers; sim3_out is the input when round 2 did
 * not run.  stats: [n_outliers_round1, then per round (iterations, trials, chi2, lambda_init, failed iteration or -1)]. */
unsigned orc_transform_optimize(int n, int fix_scale, const double* sim3_in, const double* R1, const double* t1, const double* R2, const double* t2,
                                const double* cam1, const double* cam2, const float* obs1, const float* w1, const double* pw2, const float* obs2,
                                const float* w2, const double* pw1, float chi_sq, int num_iter, double* sim3_out, uint8_t* keep, double* stats) {
    tprob_t P;
    memset(&P, 0, sizeof(P));
    P.n = n;
    P.fix_scale = fix_scale;
    t_cam(cam1, &P.c[0]);
    t_cam(cam2, &P.c[1]);
    P.obs[0] = obs1; P.w[0] = w1; P.obs[1] = obs2; P.w[1] = w2;
    P.pc[0] = (double*)malloc(sizeof(double) * (3 * (size_t)n + 1));
    P.pc[1] = (double*)malloc(sizeof(double) * (3 * (size_t)n + 1));
    for (int i = 0; i < n; ++i) {
        t_rigid(R2, t2, pw2 + 3 * i, P.pc[0] + 3 * i);
        t_rigid(R1, t1, pw1 + 3 * i, P.pc[1] + 3 * i);
        keep[i] = 1;
    }
    P.keep = keep;
    P.delta = (double)sqrtf(chi_sq);
    sim3_t cur, last;
    memcpy(&cur, sim3_in, sizeof(cur));
    last = cur;
    memcpy(sim3_out, sim3_in, sizeof(cur));
    for (int k = 0; k < 11; ++k) stats[k] = 0;
    stats[5] = stats[10] = -1;
    t_lm_round(&P, &cur, &last, 5, stats + 1);
    int bad = 0;
    for (int i = 0; i < n; ++i) {
        double e[2];
        const double c12 = t_edge_at(&last, 0, P.pc[0] + 3 * i, &P.c[0], obs1 + 2 * i, (double)w1[i], e);
        const double c21 = t_edge_at(&last, 1, P.pc[1] + 3 * i, &P.c[1], obs2 + 2 * i, (double)w2[i], e);
        if (c12 < chi_sq && c21 < chi_sq) continue;
        keep[i] = 0;
        ++bad;
    }
    stats[0] = bad;
    unsigned good = 0;
    if (n - bad >= 10) {
        t_lm_round(&P, &cur, &last, num_iter, stats + 6);
        for (int i = 0; i < n; ++i) {
            if (!keep[i]) continue;
            double e[2];
            const double c12 = t_edge_at(&last, 0, P.pc[0] + 3 * i, &P.c[0], obs1 + 2 * i, (double)w1[i], e);
            const double c21 = t_edge_at(&last, 1, P.pc[1] + 3 * i, &P.c[1], obs2 + 2 * i, (double)w2[i], e);
            if (chi_sq < c12 || chi_sq < c21) { keep[i] = 0; continue; }
            ++good;
        }
        memcpy(sim3_out, &cur, sizeof(cur));
    }
    free(P.pc[0]);
    free(P.pc[1]);
    return good;
}
