// The depth-seeded landmarks of a stereo or RGB-D keyframe on the device: the depth branch of
// module::keyframe_inserter::create_new_keyframe (module/keyframe_inserter.cc:160-212) and the landmark loop of
// module::initializer::create_map_for_stereo (module/initializer.cc:363-387) as one call of b200_depth_landmarks.  The device sorts the
// valid depths, walks them with the reference's stop and skip rules and unprojects every new landmark (data::triangulate_stereo); the
// landmark objects are then built here in the returned order, which is the order of map_database::next_landmark_id_.
//
// Call sites (USE_B200), each replacing the loop that follows the comment or test named:
//   keyframe_inserter::create_new_keyframe, after `if (!keyfrm->depth_is_available()) return keyfrm;`:
//       create_depth_landmarks_b200(map_db, curr_frm, keyfrm, B200_DEPTH_LM_KEYFRAME);
//       return keyfrm;
//     (still under the lock_guard on data::map_database::mtx_database_ the function takes at its top)
//   initializer::create_map_for_stereo, in place of the `for (unsigned int idx = 0; ...)` loop:
//       create_depth_landmarks_b200(map_db_, curr_frm, curr_keyfrm, B200_DEPTH_LM_INITIAL);
// compute_descriptor() of a landmark with one observation takes that keypoint's own descriptor, and
// update_mean_normal_and_obs_scale_variance() gives the values b200_depth_landmarks returns; both stay the landmark's own calls here
// because data::landmark keeps those members private.
#include "stella_vslam/camera/base.h"
#include "stella_vslam/camera/fisheye.h"
#include "stella_vslam/camera/perspective.h"
#include "stella_vslam/camera/radial_division.h"
#include "stella_vslam/data/frame.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/data/map_database.h"
#include "stella_vslam/feature/orb_params.h"

#include <memory>
#include <stdexcept>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace module {
namespace {

b200_matcher_t depth_landmarks_matcher() {
    static thread_local b200_matcher_t h = nullptr;
    if (!h && b200_matcher_create(0, &h) != B200_OK) throw std::runtime_error(b200_last_error());
    return h;
}

}  // namespace

unsigned int create_depth_landmarks_b200(data::map_database* map_db, data::frame& curr_frm, const std::shared_ptr<data::keyframe>& keyfrm,
                                         int mode) {
    const auto& obs = curr_frm.frm_obs_;
    const unsigned int n = obs.undist_keypts_.size();
    if (obs.depths_.size() != n) throw std::runtime_error("create_depth_landmarks_b200: the frame has no depths");
    b200_depth_landmarks_problem_t p{};
    p.mode = mode;
    const camera::base* cam = curr_frm.camera_;
    switch (cam->model_type_) {  // data/common.cc:192-260: the same members for the three perspective-family models
        case camera::model_type_t::Perspective: {
            const auto* c = static_cast<const camera::perspective*>(cam);
            p.model = 0;
            p.fx_inv = c->fx_inv_; p.fy_inv = c->fy_inv_; p.cx = c->cx_; p.cy = c->cy_;
            break;
        }
        case camera::model_type_t::Fisheye: {
            const auto* c = static_cast<const camera::fisheye*>(cam);
            p.model = 2;
            p.fx_inv = c->fx_inv_; p.fy_inv = c->fy_inv_; p.cx = c->cx_; p.cy = c->cy_;
            break;
        }
        case camera::model_type_t::RadialDivision: {
            const auto* c = static_cast<const camera::radial_division*>(cam);
            p.model = 3;
            p.fx_inv = c->fx_inv_; p.fy_inv = c->fy_inv_; p.cx = c->cx_; p.cy = c->cy_;
            break;
        }
        default:
            p.model = 1;  // equirectangular: rejected by the device when a depth is valid, as triangulate_stereo throws
    }
    p.depth_thr = keyfrm->camera_->depth_thr_;
    const Mat44_t pose_wc = curr_frm.get_pose_wc();
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) p.pose_wc[4 * r + c] = pose_wc(r, c);
    std::vector<float> x(n), y(n);
    std::vector<int32_t> octave(n);
    std::vector<uint8_t> has_landmark(n, 0);
    for (unsigned int idx = 0; idx < n; ++idx) {
        x[idx] = obs.undist_keypts_[idx].pt.x;
        y[idx] = obs.undist_keypts_[idx].pt.y;
        octave[idx] = obs.undist_keypts_[idx].octave;
        if (mode == B200_DEPTH_LM_KEYFRAME && curr_frm.get_landmark(idx)) has_landmark[idx] = 1;  // keyframe_inserter.cc:194-200
    }
    const auto* orb = curr_frm.orb_params_;
    p.n_keypoints = static_cast<int32_t>(n);
    p.x = x.data();
    p.y = y.data();
    p.octave = octave.data();
    p.depth = obs.depths_.data();
    p.has_landmark = mode == B200_DEPTH_LM_KEYFRAME ? has_landmark.data() : nullptr;
    p.num_levels = static_cast<int32_t>(orb->num_levels_);
    p.scale_factors = orb->scale_factors_.data();
    p.inv_scale_factor_last = orb->inv_scale_factors_.at(orb->num_levels_ - 1);
    std::vector<int32_t> created(n);
    std::vector<double> pos_w(3 * (size_t)n), mean_normal(3 * (size_t)n);
    std::vector<float> min_valid(n), max_valid(n);
    p.created_idx = created.data();
    p.pos_w = pos_w.data();
    p.mean_normal = mean_normal.data();
    p.min_valid_dist = min_valid.data();
    p.max_valid_dist = max_valid.data();
    if (b200_depth_landmarks(depth_landmarks_matcher(), 1, &p) != B200_OK) throw std::runtime_error(b200_last_error());
    for (int k = 0; k < p.n_created; ++k) {
        const unsigned int idx = static_cast<unsigned int>(created[k]);
        const Vec3_t pos{pos_w[3 * k], pos_w[3 * k + 1], pos_w[3 * k + 2]};
        auto lm = std::make_shared<data::landmark>(map_db->next_landmark_id_++, pos, keyfrm);
        lm->connect_to_keyframe(keyfrm, idx);
        curr_frm.add_landmark(lm, idx);
        lm->compute_descriptor();
        lm->update_mean_normal_and_obs_scale_variance();
        map_db->add_landmark(lm);
    }
    return static_cast<unsigned int>(p.n_created);
}

}  // namespace module
}  // namespace stella_vslam
