// system::create_RGBD_frame after the extraction (system.cc:467-530) on the device: undistortion, bearings and the depth of every keypoint
// in one call of b200_rgbd_depths, which reads the keypoints where the GPU extractor left them.  Only the depth map goes up; the
// reference's convert_to_true_depth of the whole map is not needed, as only the sampled pixels are converted.
//
// Call site (system::create_RGBD_frame, USE_B200): keep the grayscale conversion and extractor_left_->extract(...), drop
// util::convert_to_true_depth(img_depth, ...), and replace everything from camera_->undistort_keypoints(...) to
// camera_->convert_keypoints_to_bearings(...) with
//     rgbd_frame_b200(extractor_left_, camera_, depthmap, depthmap_factor_, frm_obs);
// `depthmap` is the caller's CV_16UC1 or CV_32FC1 map as it arrives.  Unlike the reference, which only warns, a depth map whose size
// differs from the frame is an error here (the reference would read out of bounds).
#include "stella_vslam/camera/base.h"
#include "stella_vslam/camera/fisheye.h"
#include "stella_vslam/camera/perspective.h"
#include "stella_vslam/camera/radial_division.h"
#include "stella_vslam/data/frame_observation.h"
#include "stella_vslam/feature/orb_extractor.h"

#include <opencv2/core.hpp>

#include <stdexcept>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace feature {
b200_orb_t b200_handle_of(const orb_extractor* self);  // orb_extractor_b200.cc
}

void rgbd_frame_b200(const feature::orb_extractor* extractor, const camera::base* cam, const cv::Mat& depthmap, const double depthmap_factor,
                     data::frame_observation& frm_obs) {
    const b200_orb_t orb = feature::b200_handle_of(extractor);
    if (!orb) throw std::runtime_error("rgbd_frame_b200: the extractor has not extracted a frame yet");
    b200_camera_intrinsics_t ci{};
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
            ci.model = 1;  // equirectangular: b200_rgbd_depths rejects it, as triangulate_stereo throws for RGB-D
    }
    ci.cols = cam->cols_;
    ci.rows = cam->rows_;
    const int cap = b200_orb_max_keypoints(orb, depthmap.cols, depthmap.rows);
    if (cap < 0) throw std::runtime_error(b200_last_error());
    std::vector<b200_keypoint_t> und(cap);
    std::vector<double> bearings(3 * (size_t)cap);
    std::vector<float> depths(cap), x_right(cap);
    int32_t n = 0;
    // the depth type codes are cv::Mat::type()'s (B200_DEPTH_16UC1 = CV_16UC1, B200_DEPTH_32FC1 = CV_32FC1)
    if (b200_rgbd_depths(orb, 1, &ci, cam->focal_x_baseline_, depthmap_factor, depthmap.type(), depthmap.data, depthmap.cols, depthmap.rows,
                         depthmap.step, 0, cap, und.data(), bearings.data(), depths.data(), x_right.data(), &n)
        != B200_OK)
        throw std::runtime_error(b200_last_error());
    frm_obs.undist_keypts_.resize(n);
    frm_obs.bearings_.resize(n);
    for (int i = 0; i < n; ++i) {
        cv::KeyPoint& k = frm_obs.undist_keypts_[i];  // the default cv::KeyPoint the reference's undistort_keypoints fills
        k.pt.x = und[i].x;
        k.pt.y = und[i].y;
        k.size = und[i].size;
        k.angle = und[i].angle;
        k.response = und[i].response;
        k.octave = und[i].octave;
        frm_obs.bearings_[i] = Vec3_t{bearings[3 * i], bearings[3 * i + 1], bearings[3 * i + 2]};
    }
    frm_obs.depths_.assign(depths.begin(), depths.begin() + n);
    frm_obs.stereo_x_right_.assign(x_right.begin(), x_right.begin() + n);
}

}  // namespace stella_vslam
