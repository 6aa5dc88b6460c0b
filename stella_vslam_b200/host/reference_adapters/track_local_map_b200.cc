// The GPU-shaped part of tracking_module::track_local_map as one call: tracking_module::search_local_landmarks
// (tracking_module.cc:533-606) followed by the solve of optimize_current_frame_with_local_map (:441-448), chained on the device by
// b200_track_local_map -- the frame's keypoints and descriptors are read where the GPU extractor left them, only the local map goes
// up and the landmark slots / pose / outlier flags come back.
//
// Call site (tracking_module::track_local_map, tracking_module.cc:253-275, USE_B200):
//     succeeded = search_local_landmarks(fixed_keyframe_id_threshold);            -> replaced by track_local_map_b200(...)
//     ... optimize_current_frame_with_local_map(...):  pose_optimizer_->optimize(curr_frm_, optimized_pose, outlier_flags);
//                                                                                 -> uses the pose / flags this function returned
// Precondition: `extractor` is the (left) feature::orb_extractor whose LAST extract() produced curr_frm (true in system.cc:380-395:
// one extract per frame, frame constructed from its outputs), so frame 0 of its last batch is this frame.
#include "stella_vslam/camera/base.h"
#include "stella_vslam/data/frame.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/feature/orb_extractor.h"
#include "stella_vslam/feature/orb_params.h"

#include <cstring>
#include <stdexcept>
#include <unordered_set>

#include "b200vslam.h"
#include "track_params_b200.h"

namespace stella_vslam {
namespace feature {
b200_orb_t b200_handle_of(const orb_extractor* self);  // orb_extractor_b200.cc
}

// Returns false when no local landmark is observable ("projection candidate not found", :596-599); then nothing else is touched.
// On success curr_frm carries the new landmarks (frm.add_landmark in the reference's order) and optimized_pose / outlier_flags hold
// what pose_optimizer::optimize(curr_frm, ...) would return (pose_optimizer_g2o.cc:38-175); *num_valid_obs its return value.
bool track_local_map_b200(data::frame& curr_frm, const std::vector<std::shared_ptr<data::landmark>>& local_landmarks,
                          const feature::orb_extractor* extractor, unsigned int fixed_keyframe_id_threshold, float margin,
                          Mat44_t& optimized_pose, std::vector<bool>& outlier_flags, unsigned int* num_valid_obs) {
    const b200_orb_t orb = feature::b200_handle_of(extractor);
    if (!orb) throw std::runtime_error("track_local_map_b200: the extractor has not extracted a frame yet");
    static thread_local b200_matcher_t matcher = nullptr;
    static thread_local b200_lba_t opt = nullptr;
    if (!matcher && b200_matcher_create(0, &matcher) != B200_OK) throw std::runtime_error(b200_last_error());
    if (!opt && b200_lba_create(0, &opt) != B200_OK) throw std::runtime_error(b200_last_error());

    const unsigned int num_keypts = curr_frm.frm_obs_.undist_keypts_.size();
    // ---- the landmark table: first the landmarks the frame already carries (skipped by the search, :536-551), then the local landmarks
    //      that pass the tests of :561-586, in local_landmarks_ order
    std::vector<std::shared_ptr<data::landmark>> table;
    std::vector<double> pos, nrm;
    std::vector<float> lo, hi;
    std::vector<uint8_t> desc, skip, has_obs;
    std::vector<int32_t> kp_landmark(num_keypts, -1);
    auto push = [&](const std::shared_ptr<data::landmark>& lm, uint8_t skipped) {
        const Vec3_t p = lm->get_pos_in_world(), n = lm->get_obs_mean_normal();
        pos.insert(pos.end(), {p(0), p(1), p(2)});
        nrm.insert(nrm.end(), {n(0), n(1), n(2)});
        lo.push_back(lm->get_min_valid_distance());
        hi.push_back(lm->get_max_valid_distance());
        const cv::Mat d = lm->get_descriptor();
        desc.insert(desc.end(), d.ptr<uint8_t>(), d.ptr<uint8_t>() + 32);
        skip.push_back(skipped);
        has_obs.push_back(lm->has_observation() ? 1 : 0);
        table.push_back(lm);
    };
    std::unordered_set<unsigned int> curr_landmark_ids;
    for (unsigned int idx = 0; idx < num_keypts; ++idx) {
        const auto& lm = curr_frm.get_landmark(idx);
        if (!lm || lm->will_be_erased()) continue;
        curr_landmark_ids.insert(lm->id_);
        lm->increase_num_observable();
        kp_landmark[idx] = static_cast<int32_t>(table.size());
        push(lm, 1);
    }
    const size_t first_local = table.size();
    for (const auto& lm : local_landmarks) {
        if (curr_landmark_ids.count(lm->id_) || lm->will_be_erased()) continue;
        if (fixed_keyframe_id_threshold > 0) {  // :565-585
            const auto observations = lm->get_observations();
            unsigned int temporal_observations = 0;
            for (const auto& obs : observations) {
                const auto keyfrm = obs.first.lock();
                if (keyfrm->id_ >= fixed_keyframe_id_threshold) ++temporal_observations;
            }
            if (static_cast<double>(temporal_observations) / observations.size() > 0.5) continue;
        }
        push(lm, 0);
    }

    // ---- one chain call
    b200_track_params_t prm{};
    fill_track_params(curr_frm, prm);
    prm.margin = margin;
    prm.lowe_ratio = 0.8f;     // match::projection projection_matcher(0.8), :599
    prm.hamming_thr = 100;     // HAMMING_DIST_THR_HIGH
    prm.ray_cos_thr = 0.5f;    // :588

    const Mat44_t pose_cw = curr_frm.get_pose_cw();
    double pose[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) pose[4 * r + c] = pose_cw(r, c);
    std::vector<uint8_t> observable(table.size() + 1), kp_outlier(num_keypts + 1);
    std::vector<int32_t> kp_landmark_out(num_keypts + 1, -1);
    b200_track_frame_t f{};
    f.frame = 0;
    f.pose_cw = pose;
    f.n_keypoints_in = static_cast<int32_t>(num_keypts);
    f.kp_x_right = curr_frm.frm_obs_.stereo_x_right_.empty() ? nullptr : curr_frm.frm_obs_.stereo_x_right_.data();
    f.kp_landmark = kp_landmark.data();
    f.n_landmarks = static_cast<int32_t>(table.size());
    f.lm_pos_w = pos.data(); f.lm_mean_normal = nrm.data(); f.lm_min_valid_dist = lo.data(); f.lm_max_valid_dist = hi.data();
    f.lm_desc = desc.data(); f.lm_skip = skip.data(); f.lm_has_observation = has_obs.data();
    f.kp_cap = static_cast<int32_t>(num_keypts);
    f.lm_observable = observable.data(); f.kp_landmark_out = kp_landmark_out.data(); f.kp_outlier = kp_outlier.data();
    if (b200_track_local_map(orb, matcher, opt, &prm, 1, &f) != B200_OK) throw std::runtime_error(b200_last_error());
    if (static_cast<unsigned int>(f.n_keypoints) != num_keypts) throw std::runtime_error("track_local_map_b200: the extractor's last frame is not curr_frm");

    // ---- write-back in the reference's order
    bool found_proj_candidate = false;
    for (size_t l = first_local; l < table.size(); ++l)
        if (observable[l]) {
            table[l]->increase_num_observable();  // :594
            found_proj_candidate = true;
        }
    if (!found_proj_candidate) return false;  // (the reference returns before matching and optimising; curr_frm is unchanged)
    for (unsigned int idx = 0; idx < num_keypts; ++idx) {
        const int32_t l = kp_landmark_out[idx];
        if (l >= static_cast<int32_t>(first_local) && l != kp_landmark[idx]) curr_frm.add_landmark(table[l], idx);  // projection.cc:87
    }
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) optimized_pose(r, c) = f.pose_cw_out[4 * r + c];
    outlier_flags.assign(num_keypts, false);
    for (unsigned int idx = 0; idx < num_keypts; ++idx) outlier_flags[idx] = kp_outlier[idx] != 0;
    if (num_valid_obs) *num_valid_obs = f.n_valid;
    return true;
}

}  // namespace stella_vslam
