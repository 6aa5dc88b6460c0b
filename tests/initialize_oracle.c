/* initialize_oracle.c -- CPU restatement of the reconstruction of initialize::perspective / initialize::bearing_vector
 * (src/stella_vslam/initialize/base.cc, perspective.cc:83-126, bearing_vector.cc:58-77): the H / F / E decompositions, base::triangulate
 * for every hypothesis and base::find_most_plausible_pose.  The arithmetic is stella_vslam_b200/csrc/initialize_core.h compiled as C here
 * (-ffp-contract=off), on twoview_oracle.c's pieces, with tests/motion_track_oracle.c's reproject_to_image; the loop over the matches,
 * the sort of the parallax cosines and the selection follow base.cc directly.  The RANSAC stage is twoview_oracle.c's and
 * essential_oracle.c's, composed by tests/initialize_oracle.py.  Test infrastructure, compiled on first use. */
#include "twoview_oracle.c"

void mto_reproject(int model, double fx, double fy, double cx, double cy, double fxb, double cols, double rows, const float* bounds, const double* Rt_cw,
                   int n, const double* pos_w, uint8_t* in_image, double* reproj, float* x_right);

/* model, fx, fy, cx, cy, cols, rows, then the float bounds */
typedef struct {
    int model;
    double fx, fy, cx, cy, cols, rows;
    float bounds[4];
} in_cam_t;

static int in_reproject(const in_cam_t* c, const double* Rt, const double* p, double* q) {
    uint8_t vis;
    float xr;
    mto_reproject(c->model, c->fx, c->fy, c->cx, c->cy, 0.0, c->cols, c->rows, c->bounds, Rt, 1, p, &vis, q, &xr);
    return vis;
}

#define IN_FSQRT(x) sqrtf(x)
#include "../stella_vslam_b200/csrc/initialize_core.h"

static in_cam_t make_cam(const double* c) {
    in_cam_t r;
    r.model = (int)c[0];
    r.fx = c[1], r.fy = c[2], r.cx = c[3], r.cy = c[4], r.cols = c[5], r.rows = c[6];
    for (int k = 0; k < 4; ++k) r.bounds[k] = (float)c[7 + k];
    return r;
}

int ino_choose_H(float cost_H, float cost_F, int valid_H) { return in_choose_H(cost_H, cost_F, valid_H); }

int ino_svd33(const double* A, double* U, double* s, double* V) { return in_svd33(A, U, s, V); }

int ino_decompose_H(const double* H, const double* K1, const double* K2, double* R, double* t, double* nrm, int* status) {
    *status = 0;
    return in_decompose_H(H, K1, K2, R, t, nrm, status);
}

int ino_decompose_E(const double* E, double* R, double* t) {
    int status = 0;
    in_decompose_E(E, R, t, &status);
    return status;
}

void ino_essential_of_F(const double* F, const double* K1, const double* K2, double* E) { in_essential_of_F(F, K1, K2, E); }

void ino_midpoint(const double* b1, const double* b2, const double* R, const double* t, double* p) { in_midpoint(b1, b2, R, t, p); }

static int cmp_float(const void* a, const void* b) {
    const float x = *(const float*)a, y = *(const float*)b;
    return x < y ? -1 : (y < x ? 1 : 0);
}

/* base::triangulate(R, t, is_inlier_match, depth_is_positive) over the n matches (ref index, cur index).  cams: 11 doubles per view
 * (model fx fy cx cy cols rows bounds[4]).  Out: pts (n_ref x 3, zeros where not triangulated), flags (n_ref), *num_triangulated,
 * *parallax_cos.  Returns nums_valid. */
int ino_triangulate(const double* cams, const double* Rt, int depth_is_positive, float reproj_err_thr, int n_ref, const float* undist_ref,
                    const double* bearings_ref, const float* undist_cur, const double* bearings_cur, int n, const int32_t* matches,
                    const uint8_t* inlier, double* pts, uint8_t* flags, int* num_triangulated, float* parallax_cos) {
    const in_cam_t cr = make_cam(cams), cc = make_cam(cams + 11);
    const float thr_sq = reproj_err_thr * reproj_err_thr;
    double ctr[3];
    in_neg_rt_t(Rt, Rt + 9, ctr);
    float* cosp = (float*)malloc(sizeof(float) * (size_t)(n > 0 ? n : 1));
    memset(pts, 0, sizeof(double) * 3 * (size_t)n_ref);
    memset(flags, 0, (size_t)n_ref);
    int n_valid = 0, n_tri = 0;
    for (int j = 0; j < n; ++j) {
        if (!inlier[j]) continue;
        const int kr = matches[2 * j], kc = matches[2 * j + 1];
        double p[3];
        float c;
        const int s = in_match(&cr, &cc, Rt, ctr, depth_is_positive, thr_sq, bearings_ref + 3 * (size_t)kr, bearings_cur + 3 * (size_t)kc,
                               undist_ref + 2 * (size_t)kr, undist_cur + 2 * (size_t)kc, p, &c);
        if (s == IN_TRI_REJECTED) continue;
        cosp[n_valid++] = c;
        if (s == IN_TRI_TRIANGULATED) {
            memcpy(pts + 3 * (size_t)kr, p, sizeof p);
            flags[kr] = 1;
            ++n_tri;
        }
    }
    if (n_valid > 0) {
        qsort(cosp, (size_t)n_valid, sizeof(float), cmp_float);
        *parallax_cos = cosp[n_valid - 1 < 50 ? n_valid - 1 : 50];
    } else {
        *parallax_cos = 1.0f;
    }
    *num_triangulated = n_tri;
    free(cosp);
    return n_valid;
}

int ino_select(int n_hyp, const int32_t* nums_valid, const int32_t* num_triangulated, const float* parallax_cos, uint32_t min_valid, uint32_t min_tri,
               double cos_thr, int* best) {
    return in_select(n_hyp, nums_valid, num_triangulated, parallax_cos, min_valid, min_tri, cos_thr, best);
}

/* reconstruct_with_H / _F / _E (model IN_MODEL_*) from the solver's matrix M and inlier flags: the decomposition, every hypothesis'
 * triangulation and find_most_plausible_pose.  Out as b200_init_problem_t: stage, n_hyp, per hypothesis nums_valid, num_triangulated,
 * parallax_cos, and (when find_most_plausible_pose ran) R / t, and on success pts / flags (n_ref).  Returns the status bits. */
int ino_reconstruct(int model, const double* M, const double* cams, const double* K1, const double* K2, uint32_t min_num_triangulated,
                    uint32_t min_num_valid_pts, double cos_thr, float reproj_err_thr, int n_ref, const float* undist_ref, const double* bearings_ref,
                    const float* undist_cur, const double* bearings_cur, int n, const int32_t* matches, const uint8_t* inlier, int* stage,
                    int* n_hyp_out, int32_t* nums_valid, int32_t* num_tri, float* parallax_cos, double* R_out, double* t_out, double* pts_out,
                    uint8_t* flags_out) {
    int status = 0, n_hyp = 0;
    double R[8 * 9], t[8 * 3];
    *n_hyp_out = 0;
    if (model == IN_MODEL_H) {
        double nrm[8 * 3];
        if (!in_decompose_H(M, K1, K2, R, t, nrm, &status)) {
            *stage = IN_STAGE_DECOMPOSE;
            return status;
        }
        n_hyp = 8;
    } else {
        double E[9];
        if (model == IN_MODEL_F) in_essential_of_F(M, K1, K2, E);
        else memcpy(E, M, sizeof E);
        in_decompose_E(E, R, t, &status);
        n_hyp = 4;
    }
    *n_hyp_out = n_hyp;
    double* pts = (double*)malloc(sizeof(double) * 3 * 8 * (size_t)(n_ref > 0 ? n_ref : 1));
    uint8_t* fl = (uint8_t*)malloc(8 * (size_t)(n_ref > 0 ? n_ref : 1));
    for (int h = 0; h < n_hyp; ++h) {
        double Rt[12];
        memcpy(Rt, R + 9 * h, 9 * sizeof(double));
        memcpy(Rt + 9, t + 3 * h, 3 * sizeof(double));
        nums_valid[h] = ino_triangulate(cams, Rt, model != IN_MODEL_E, reproj_err_thr, n_ref, undist_ref, bearings_ref, undist_cur, bearings_cur, n,
                                        matches, inlier, pts + 3 * (size_t)h * n_ref, fl + (size_t)h * n_ref, &num_tri[h], &parallax_cos[h]);
    }
    int best;
    *stage = in_select(n_hyp, nums_valid, num_tri, parallax_cos, min_num_valid_pts, min_num_triangulated, cos_thr, &best);
    const int ok = *stage == IN_STAGE_SUCCEEDED;
    for (int k = 0; k < 9; ++k) R_out[k] = ok ? R[9 * best + k] : 0.0;
    for (int k = 0; k < 3; ++k) t_out[k] = ok ? t[3 * best + k] : 0.0;
    if (ok) {
        memcpy(pts_out, pts + 3 * (size_t)best * n_ref, sizeof(double) * 3 * (size_t)n_ref);
        memcpy(flags_out, fl + (size_t)best * n_ref, (size_t)n_ref);
    }
    free(pts);
    free(fl);
    return status;
}
