/*
 * oracle/oracle.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the stella_vslam hot path (ORB extract -> Hamming match -> local BA).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 * Every function cites the reference file:line it follows (paths relative to the reference checkout).
 * Third-party arithmetic that is NOT in the reference tree (OpenCV 4.x cv::resize / cv::FAST /
 * cv::GaussianBlur / cv::fastAtan2, g2o 20230223_git LM + Schur) is restated from the published
 * algorithms; the OpenCV pieces are pinned bit-for-bit against cv2 4.13.0 by tests/golden (see
 * tests/golden/make_golden.py), the g2o piece is "parity unpinned" (see oracle/lba_oracle.c header).
 */
#ifndef B200VSLAM_ORACLE_H
#define B200VSLAM_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* cv::KeyPoint fields the reference fills (class_id stays -1). */
typedef struct {
    float x, y, size, angle, response;
    int32_t octave;
} orc_keypoint_t;

/* feature::orb_params (orb_params.cc:12-27) + orb_extractor ctor's min_area (orb_extractor.cc:16-20). */
typedef struct {
    float scale_factor;    /* 1.2 */
    int32_t num_levels;    /* 8 */
    int32_t ini_fast_thr;  /* 20 */
    int32_t min_fast_thr;  /* 7 */
    uint32_t min_area;     /* Preprocessing.min_size, system.cc:95 (default 800) */
} orc_orb_config_t;

/* ---- ORB primitives -------------------------------------------------------------------------- */
void orc_scale_factors(float scale_factor, int n, float* sf, float* inv_sf, float* sigma_sq, float* inv_sigma_sq);
void orc_level_size(int w, int h, float sf, int* lw, int* lh);
void orc_resize_linear_u8(const uint8_t* src, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh, int dstride);
int orc_fast9_16_nms(const uint8_t* img, int stride, int w, int h, int thr, int16_t* xs, int16_t* ys, uint8_t* scores, int cap);
void orc_gaussian7_s2_u8(const uint8_t* src, int w, int h, int sstride, uint8_t* dst, int dstride);
float orc_fast_atan2(float y, float x);
float orc_ic_angle(const uint8_t* img, int stride, int x, int y);
float orc_util_cos(float v);
float orc_util_sin(float v);
void orc_rbrief(const uint8_t* blurred, int stride, float x, float y, float angle_deg, uint8_t* desc32);
void orc_rect_mask(int cols, int rows, const float* rects, int n_rects, uint8_t* mask, int mstride);

/* feature::orb_extractor::extract (orb_extractor.cc:28-136).  Returns N (>=0), or -1 if cap is too small.
 * level_counts / raw_counts: optional [num_levels] outputs (kept keypoints, raw FAST candidates).
 * pyramid_out: optional array of num_levels caller buffers (tight stride = level width) receiving image_pyramid_. */
int orc_orb_extract(const uint8_t* img, int w, int h, int stride, const uint8_t* mask, int mask_stride,
                    const orc_orb_config_t* cfg, orc_keypoint_t* kps, uint8_t* descs, int cap, int* level_counts,
                    int* raw_counts, uint8_t** pyramid_out);

void orc_convert_to_grayscale(const uint8_t* src, int w, int h, int stride, int channels, int rgb_order, uint8_t* dst, int dstride);

/* ---- matchers --------------------------------------------------------------------------------- */
unsigned orc_hamming_32(const uint8_t* a, const uint8_t* b);
unsigned orc_hamming_64(const uint8_t* a, const uint8_t* b);
float orc_angle_diff(float a1, float a2);
/* match::robust::brute_force_match (match/robust.cc:232-328).  valid2[i]!=0 <=> keyframe keypoint i has a live
 * landmark.  pairs_out: (idx_1, idx_2) sorted by idx_1.  Returns the number of matches. */
int orc_brute_force_match(const uint8_t* desc1, const float* angle1, int n1, const uint8_t* desc2, const float* angle2,
                          const uint8_t* valid2, int n2, float lowe_ratio, int check_orientation, int32_t* pairs_out);

/* data::landmark::compute_descriptor (data/landmark.cc:199-256): index of the representative descriptor among n x 32 bytes. */
int orc_landmark_descriptor(const uint8_t* descs, int n);

/* ---- grid-guided projection matchers (guided_oracle.c) ------------------------------------------------------------ */
typedef struct {
    int32_t n_train;                 /* frame keypoints (the side that is searched) */
    const float* t_x;                /* undist_keypts_[i].pt.x */
    const float* t_y;
    const uint8_t* t_octave;
    const float* t_angle;            /* may be NULL when orientation is not checked */
    const float* t_x_right;          /* frm_obs_.stereo_x_right_ or NULL when empty */
    const uint8_t* t_desc;           /* N x 32 */
    uint8_t* t_occupied;             /* N, in/out: keypoint already carries a landmark with observations */
    float min_x, max_x, min_y, max_y; /* camera->img_bounds_ */
    int32_t grid_cols, grid_rows;    /* num_grid_cols_/rows_ (64 x 48) */
    int32_t n_queries;               /* landmarks, in the reference's iteration order */
    const uint8_t* q_desc;           /* Q x 32 (landmark::get_descriptor) */
    const float* q_x;                /* reprojection */
    const float* q_y;
    const float* q_margin;           /* margin * scale_factors_[level] (float product) */
    const int8_t* q_min_level;       /* < 0: unchecked */
    const int8_t* q_max_level;
    const float* q_x_right;          /* reprojected x_right (used when t_x_right != NULL) */
    const float* q_angle;            /* mode 1 */
    const uint8_t* q_valid;          /* 0: skipped before the search (not reprojected / will_be_erased / outside the image); NULL = all */
    const uint8_t* q_has_observation; /* modes 0 / 1: landmark::has_observation(); NULL = all (projection.cc:50-53, 163-166) */
    const double* q_reproj;          /* mode 3: Q x 2 reprojection in double (fuse.cc:96-97) */
    const float* inv_level_sigma_sq; /* mode 3: orb_params_->inv_level_sigma_sq_ */
    int32_t do_reprojection_matching; /* mode 3 */
} orc_guided_t;
/* mode 0: projection::match_frame_and_landmarks (projection.cc:13-93); mode 1: match_current_and_last_frames (:95-207),
 * match_frame_and_keyframe (:217-319), match_by_Sim3_transform (:321-416); mode 2: one direction of match_keyframes_mutually
 * (:418-630, stateless); mode 3: fuse::detect_duplication (fuse.cc:12-154); mode 4: area::match_in_consistent_area (area.cc:8-98).
 * match_out[q] = frame keypoint index or -1.  Returns the number of matches. */
int orc_match_guided(const orc_guided_t* P, int mode, unsigned thr, float lowe_ratio, int check_orientation, int32_t* match_out);
int orc_cross_check(const int32_t* idx2_in_1, int n1, const int32_t* idx1_in_2, int n2, int32_t* mutual_out);

/* ---- match::stereo (stereo_oracle.c): stereo::compute (stereo.cc:20-114).  pyr_*[l]: level l, tight stride = widths[l].
 * Returns the number of keypoints that keep a stereo match. */
int orc_stereo_compute(const uint8_t* const* pyr_left, const uint8_t* const* pyr_right, const int* widths, const int* heights,
                       const orc_keypoint_t* kl, const uint8_t* dl, int n_left, const orc_keypoint_t* kr, const uint8_t* dr, int n_right,
                       const float* scale_factors, const float* inv_scale_factors, float focal_x_baseline, float true_baseline,
                       float* stereo_x_right, float* depths);

/* ---- per-keypoint steps between extractor and matchers (camera_oracle.c) --------------------------------------------------- */
void orc_undistort_points(const float* xy_in, int n, double fx, double fy, double cx, double cy, const double* dist5, int max_iter, double eps,
                          float* xy_out);
void orc_points_to_bearings(const float* xy, int n, int model, double fx, double fy, double cx, double cy, double cols, double rows,
                            double* bearings);

void orc_can_observe(int model, double fx, double fy, double cx, double cy, double fxb, double cols, double rows, const float* bounds,
                     const double* Rt_cw, const double* trans_wc, int n, const double* pos_w, const double* mean_normal,
                     const float* min_valid_dist, const float* max_valid_dist, float ray_cos_thr, unsigned num_levels, float log_scale_factor,
                     uint8_t* observable, double* reproj, float* x_right, uint32_t* pred_scale_level);

void orc_landmark_geometry(int n, const double* pos_w, const int32_t* offsets, const double* cam_centers, const double* ref_center,
                           const float* ref_scale_factor, float inv_scale_factor_last, double* mean_normal, float* max_valid_dist,
                           float* min_valid_dist);

/* ---- all-pairs matchers with greedy state (pairs_oracle.c) ------------------------------------------------------------ */
typedef struct {
    int32_t n1;                  /* rows: keyframe 1 / the keyframe */
    const uint8_t* desc1;
    const float* angle1;
    const uint8_t* valid1;       /* row takes part (BOW: live landmark; TRIANGULATION: no landmark yet); NULL = all */
    const int32_t* node1;        /* BoW node id per keypoint or NULL */
    const double* bearing1;      /* TRIANGULATION: n1 x 3 */
    const float* scale1;         /* TRIANGULATION: scale_factors_[octave] per row */
    const uint8_t* stereo1;      /* TRIANGULATION: stereo_x_right_ >= 0, or NULL */
    int32_t n2;                  /* candidates: keyframe 2 / the frame */
    const uint8_t* desc2;
    const float* angle2;
    const uint8_t* valid2;
    const int32_t* node2;
    const double* bearing2;
    const uint8_t* stereo2;
    double E_12[9];              /* row-major */
    double epiplane_in_2[3];
    int32_t valid_epiplane;
    float residual_rad_thr;
} orc_pairs_t;
int orc_check_epipolar_constraint(const double* b1, const double* b2, const double* E, float residual_rad_thr, float scale_factor);
/* variant 0: bow_tree::match_frame_and_keyframe / match_keyframes; 1: robust:: / bow_tree::match_for_triangulation.
 * match_out[i] = matched candidate or -1 per row.  Returns the number of matches. */
int orc_match_pairs(const orc_pairs_t* P, int variant, float lowe_ratio, int check_orientation, int32_t* match_out);

/* ---- local bundle adjustment (lba_oracle.c; PARITY UNPINNED, see its header) ------------------------------------- */
typedef struct {
    int32_t model;            /* 0: perspective-family edges (Perspective/Fisheye/RadialDivision, reproj_edge_wrapper.h:64-188), 1: equirectangular */
    double fx, fy, cx, cy;    /* perspective */
    double fxb;               /* focal_x_baseline_ (stereo rows) */
    double cols, rows;        /* equirectangular */
} orc_camera_t;

typedef struct {
    int32_t n_poses, n_points, n_edges, n_cams;
    const double* pose_cw;          /* K x 16, row-major 4x4 (keyfrm->get_pose_cw()) */
    const uint8_t* pose_fixed;      /* K: fixed keyframes (local_bundle_adjuster_g2o.cc:184-190) */
    const double* points;           /* L x 3 (pos_w) */
    const uint8_t* point_fixed;     /* L or NULL (marker corners with keep_fixed_) */
    const int32_t* e_pose;          /* E */
    const int32_t* e_point;         /* E */
    const uint8_t* e_cam;           /* E: camera index */
    const float* e_obs;             /* E x 3: undist x, y, x_right (x_right < 0 => monocular edge) */
    const float* e_inv_sigma_sq;    /* E: inv_level_sigma_sq_[octave] */
    const float* e_delta;           /* E: Huber delta (sqrt chi-square, float) */
    const uint8_t* e_robust;        /* E or NULL(=1): Huber kernel in the first round (marker edges of fixed markers: 0) */
    const uint8_t* e_can_be_outlier;/* E or NULL(=1): landmark edges 1, marker-corner edges 0 */
    const orc_camera_t* cams;
} orc_lba_problem_t;

typedef struct {
    int32_t iterations[2];
    int32_t n_outliers;
    double chi2[2];           /* active robust chi2 after each round */
    double lambda_init;
    double lambda_final[2];
} orc_lba_stats_t;

/* local_bundle_adjuster_g2o::optimize steps 5-8 (local_bundle_adjuster_g2o.cc:306-409) on a flattened problem.
 * Returns 0, or 1 when *force_stop was already set (no write-back, :308-310). */
int orc_lba_solve(const orc_lba_problem_t* P, int iters1, int iters2, volatile uint8_t* force_stop, double* pose_cw_out,
                  double* points_out, uint8_t* outlier_out, orc_lba_stats_t* stats);
int orc_global_ba_solve(const orc_lba_problem_t* P, int num_iter, double gain_threshold, volatile uint8_t* force_stop, double* pose_cw_out,
                        double* points_out, orc_lba_stats_t* stats);
/* Test infrastructure: what build_system uses for every active edge at the state (pose_cw K x 16, points L x 3; NULL = the problem's):
 * residual (E x 3), robust weight inv_sigma_sq * rho' (E), landmark Jacobian (E x 3x3) and pose Jacobian (E x 3x6, rotation first),
 * rows past the edge's dimension and inactive edges (level[e] != 0) zero.  robust: per-edge Huber switch (NULL = P->e_robust).
 * Returns the number of active edges. */
int orc_lba_linearize(const orc_lba_problem_t* P, const double* pose_cw, const double* points, const uint8_t* level, const uint8_t* robust,
                      double* err_out, double* weight_out, double* Ji_out, double* Jj_out);

/* optimize::pose_optimizer_g2o::optimize (pose_optimizer_g2o.cc:38-175): motion-only BA of one frame.  P: one free pose, fixed
 * points, one edge per observation.  Returns the number of inlier observations; outlier_flags[e] per edge. */
unsigned orc_pose_optimize(const orc_lba_problem_t* P, int num_trials_robust, int num_trials, int num_each_iter, double* pose_cw_out,
                           uint8_t* outlier_flags);

/* timed CPU baseline driver (batch_oracle.c): n frames on n_threads pthreads, extract then match to predecessor */
int orc_frontend_batch(const uint8_t* frames, int n_unique, int n, int w, int h, const orc_orb_config_t* cfg, int cap, float lowe,
                       int check_ori, int n_threads, int* counts, int* n_matches);

#ifdef __cplusplus
}
#endif
#endif
