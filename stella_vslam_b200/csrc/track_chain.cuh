// track_chain.cuh -- internal interfaces of b200_track_local_map, b200_motion_based_track and b200_robust_match_based_track
// (include/b200vslam.h): the chains are driven from match_kernels.cu, stage A (undistort + bearings, can_observe or the last-frame
// reprojection + query build) lives in orb_kernels.cu (same device functions and -fmad=false as the stage-by-stage ABI), stage C (edge
// build + pose optimisation) in lba_kernels.cu, the robust chain's minimal-set sampler in random_array.cu and its RANSAC in
// essential_kernels.cu (essential_ransac.cuh).  Plain device pointers, no handles' internals cross a TU.
#pragma once

#include <cmath>

#include "common.cuh"

namespace b200 {
namespace chain {

// The camera models of b200_camera_intrinsics_t: 0 perspective, 1 equirectangular, 2 fisheye, 3 radial division.  Models 2 and 3 need
// finite intrinsics and coefficients (models 0 and 1 are accepted as before, whatever their values).
inline bool camera_valid(const b200_camera_intrinsics_t& c) {
    if (c.model < 0 || c.model > 3) return false;
    if (c.model < 2) return true;
    const bool coeffs = c.model == 2 ? (std::isfinite(c.k1) && std::isfinite(c.k2) && std::isfinite(c.k3) && std::isfinite(c.k4))
                                     : std::isfinite(c.distortion);
    return coeffs && std::isfinite(c.fx) && std::isfinite(c.fy) && std::isfinite(c.cx) && std::isfinite(c.cy);
}

struct TrackShared {  // by-value kernel parameter
    int model;
    double fx, fy, cx, cy, k1, k2, p1, p2, k3, cols, rows, fxb, k4, distortion;
    float min_x, max_x, min_y, max_y;
    float ray_cos_thr, log_scale_factor, margin, delta;
    unsigned num_levels;
    float scale_factors[32], inv_level_sigma_sq[32];
    // b200_motion_based_track: projection.cc:108-116
    int monocular;
    double true_baseline;
};

struct TrackFrameDev {  // one frame; every pointer is a device pointer
    // the extractor's results for this frame
    const b200_keypoint_t* kps;
    const int* n_kp;
    int kp_cap;
    // caller inputs
    int n_kp_in, n_lm;
    const float* kp_x_right;   // may be null
    const int* kp_landmark;    // may be null
    const double *pos_w, *mean_normal;
    const float *min_d, *max_d;
    const unsigned char *lm_skip, *lm_has_obs;  // may be null
    double Rt[12], twc[3];
    // stage A
    b200_keypoint_t* undist;
    float *t_x, *t_y;
    unsigned char *t_octave, *occupied;
    unsigned char* observable;
    float *q_x, *q_y, *q_margin, *q_xr;
    signed char *q_lo, *q_hi;
    unsigned char* q_valid;
    // stage B (guided matcher)
    const int* match_out;
    // stage C
    int* kp_landmark_out;
    unsigned char* kp_outlier;
    int* status;  // [0] keypoint count, [1] != 0: n_kp_in disagrees with the extractor's count, [2] edges of stage C
    // b200_motion_based_track only (null / unused in the local-map chain)
    float* t_angle;                   // stage A: angle of every keypoint, for the orientation gate
    const unsigned char* lm_octave;   // last-frame table: octave of the last frame's keypoint
    double last_Rt[12];               // last frame: rot_cw row-major, then trans_cw
    // b200_robust_match_based_track only (null in the other chains)
    double* bearings;                 // stage A: bearing of every keypoint (3 doubles)
    int* count_out;                   // stage A: the keypoint count again, in the per-frame array the brute-force matcher reads
};

// orb_kernels.cu: device views of the extractor's last batch + the stream its work is ordered on
int orb_results(b200_orb_t orb, const b200_keypoint_t** d_kps, const unsigned char** d_descs, const int** d_counts, int* stride, int* batch,
                cudaStream_t* stream, int* device);
int track_stage_a(cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, int n_frames, int max_kp, int max_lm);
// the same keypoint kernel (with t_angle), then one query per last-frame table entry (projection.cc:95-160)
int motion_stage_a(cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, int n_frames, int max_kp, int max_lm);
// the same keypoint kernel with the bearings and count_out (camera::base::convert_keypoints_to_bearings after the undistortion)
int robust_stage_a(cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, int n_frames, int max_kp);
// random_array.cu: for every problem p with d_n[p] >= set_size (<= rnd::kMaxDeviceSet), max_num_iter calls of
// util::create_random_array(set_size, 0, d_n[p] - 1) from engine p (d_engines null: default-constructed engines) into
// d_out + p * max_num_iter * set_size.  One warp per problem.
int draw_min_sets(cudaStream_t st, int n_problems, const b200_mt19937_t* d_engines, const int* d_n, uint32_t set_size, uint32_t max_num_iter,
                  int32_t* d_out);
// lba_kernels.cu: builds one edge per keypoint that carries a landmark (keypoint order), runs pose_optimizer::optimize for every frame and
// scatters the flags back to keypoint indexing.  h_frames = the host copy of d_frames; pose_out / n_valid are device pointers.
// d_gate: null, or per frame 0 = apply the matches but build no edge (the pose stays, no flag is set).
int track_stage_c(b200_lba_t opt, cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, const TrackFrameDev* h_frames,
                  const double* const* pose_cw, int n_frames, int max_kp, int trials_robust, int trials, int each_iter, double* d_pose_out,
                  unsigned* d_n_valid, cudaEvent_t ev_edges_done, const int* d_gate = nullptr);

}  // namespace chain
}  // namespace b200
