// b200_track_params_t of a frame, shared by the tracking adapters (track_local_map_b200.cc, frame_tracker_b200.cc): the camera, image
// bounds, grid, levels and pose-optimiser trials of curr_frm.  margin, lowe_ratio, hamming_thr and ray_cos_thr are each caller's.
#pragma once

#include "stella_vslam/camera/base.h"
#include "stella_vslam/camera/fisheye.h"
#include "stella_vslam/camera/perspective.h"
#include "stella_vslam/camera/radial_division.h"
#include "stella_vslam/data/frame.h"
#include "stella_vslam/feature/orb_params.h"

#include "b200vslam.h"

namespace stella_vslam {

// b200_camera_intrinsics_t and image bounds (min_x, max_x, min_y, max_y) of a camera, shared with the initialiser's adapter
// (initialize_b200.cc).  Model codes: 0 perspective, 1 equirectangular, 2 fisheye, 3 radial division (the double members; the fisheye
// undistortion rounds them to float on the device as cv_cam_matrix_ / cv_dist_params_ do).
inline void fill_camera_intrinsics(const camera::base* cam, b200_camera_intrinsics_t& ci, float* img_bounds) {
    switch (cam->model_type_) {
        case camera::model_type_t::Perspective: {
            const auto* p = static_cast<const camera::perspective*>(cam);
            ci.model = 0;
            ci.fx = p->fx_; ci.fy = p->fy_; ci.cx = p->cx_; ci.cy = p->cy_;
            ci.k1 = p->k1_; ci.k2 = p->k2_; ci.p1 = p->p1_; ci.p2 = p->p2_; ci.k3 = p->k3_;
            break;
        }
        case camera::model_type_t::Fisheye: {
            const auto* p = static_cast<const camera::fisheye*>(cam);
            ci.model = 2;
            ci.fx = p->fx_; ci.fy = p->fy_; ci.cx = p->cx_; ci.cy = p->cy_;
            ci.k1 = p->k1_; ci.k2 = p->k2_; ci.k3 = p->k3_; ci.k4 = p->k4_;
            break;
        }
        case camera::model_type_t::RadialDivision: {
            const auto* p = static_cast<const camera::radial_division*>(cam);
            ci.model = 3;
            ci.fx = p->fx_; ci.fy = p->fy_; ci.cx = p->cx_; ci.cy = p->cy_;
            ci.distortion = p->distortion_;
            break;
        }
        default:
            ci.model = 1;  // equirectangular
            break;
    }
    ci.cols = cam->cols_;
    ci.rows = cam->rows_;
    img_bounds[0] = cam->img_bounds_.min_x_; img_bounds[1] = cam->img_bounds_.max_x_;
    img_bounds[2] = cam->img_bounds_.min_y_; img_bounds[3] = cam->img_bounds_.max_y_;
}

inline void fill_track_params(const data::frame& curr_frm, b200_track_params_t& prm) {
    const auto* cam = curr_frm.camera_;
    fill_camera_intrinsics(cam, prm.cam, prm.img_bounds);
    prm.focal_x_baseline = cam->focal_x_baseline_;
    prm.monocular = cam->setup_type_ == camera::setup_type_t::Monocular ? 1 : 0;
    prm.grid_cols = static_cast<int32_t>(curr_frm.frm_obs_.num_grid_cols_);
    prm.grid_rows = static_cast<int32_t>(curr_frm.frm_obs_.num_grid_rows_);
    const auto* op = curr_frm.orb_params_;
    prm.num_levels = op->num_levels_;
    prm.log_scale_factor = op->log_scale_factor_;
    prm.scale_factors = op->scale_factors_.data();
    prm.inv_level_sigma_sq = op->inv_level_sigma_sq_.data();
    prm.num_trials_robust = 2; prm.num_trials = 2; prm.num_each_iter = 10;  // pose_optimizer_factory.h:18-47
}

}  // namespace stella_vslam
