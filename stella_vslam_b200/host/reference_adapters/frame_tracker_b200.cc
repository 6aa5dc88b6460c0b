// module::frame_tracker::motion_based_track (module/frame_tracker.cc:20-59) as one device call: the last frame's landmarks are projected
// into curr_frm, matched (a second time at twice the margin when short), the pose optimised and the outliers discarded by
// b200_motion_based_track -- the frame's keypoints and descriptors are read where the GPU extractor left them, only the last-frame table
// goes up and the landmark slots / pose come back.
//
// Call site (tracking_module::track_current_frame, tracking_module.cc:333-355, USE_B200):
//     succeeded = frame_tracker_.motion_based_track(curr_frm_, last_frm_, twist_);
//         -> succeeded = motion_based_track_b200(curr_frm_, last_frm_, twist_, extractor_left_, margin_last_frame_projection_,
//                                                num_matches_thr);
// The landmarks curr_frm now carries are the ones track_local_map_b200 (track_local_map_b200.cc) then finds in its kp_landmark table:
// they are skipped by the local-map search and become edges of its pose optimisation, as in the reference.
// Precondition: `extractor` is the (left) feature::orb_extractor whose LAST extract() produced curr_frm (true in system.cc:380-395:
// one extract per frame, frame constructed from its outputs), so frame 0 of its last batch is this frame.
#include "stella_vslam/camera/base.h"
#include "stella_vslam/data/frame.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/feature/orb_extractor.h"
#include "stella_vslam/feature/orb_params.h"

#include <cstring>
#include <random>
#include <stdexcept>

#include "b200vslam.h"
#include "pairs_gather_b200.h"
#include "track_params_b200.h"

namespace stella_vslam {
namespace feature {
b200_orb_t b200_handle_of(const orb_extractor* self);  // orb_extractor_b200.cc
}

// Returns what frame_tracker::motion_based_track returns.  curr_frm leaves with the predicted pose velocity * last pose and the matches
// of the last search when tracking failed before the pose optimisation, else with the optimised pose and the inlier landmarks.
bool motion_based_track_b200(data::frame& curr_frm, const data::frame& last_frm, const Mat44_t& velocity, const feature::orb_extractor* extractor,
                             float margin, unsigned int num_matches_thr) {
    const b200_orb_t orb = feature::b200_handle_of(extractor);
    if (!orb) throw std::runtime_error("motion_based_track_b200: the extractor has not extracted a frame yet");
    static thread_local b200_matcher_t matcher = nullptr;
    static thread_local b200_lba_t opt = nullptr;
    if (!matcher && b200_matcher_create(0, &matcher) != B200_OK) throw std::runtime_error(b200_last_error());
    if (!opt && b200_lba_create(0, &opt) != B200_OK) throw std::runtime_error(b200_last_error());

    // ---- the last-frame table: keypoints of last_frm with a landmark that is not will_be_erased, in keypoint order (projection.cc:120-128)
    const auto& last_kps = last_frm.frm_obs_.undist_keypts_;
    std::vector<std::shared_ptr<data::landmark>> table;
    std::vector<double> pos;
    std::vector<uint8_t> desc, octave, has_obs;
    std::vector<float> angle;
    for (unsigned int idx = 0; idx < last_kps.size(); ++idx) {
        const auto& lm = last_frm.get_landmark(idx);
        if (!lm || lm->will_be_erased()) continue;
        const Vec3_t p = lm->get_pos_in_world();
        pos.insert(pos.end(), {p(0), p(1), p(2)});
        const cv::Mat d = lm->get_descriptor();
        desc.insert(desc.end(), d.ptr<uint8_t>(), d.ptr<uint8_t>() + 32);
        octave.push_back(static_cast<uint8_t>(last_kps[idx].octave));
        angle.push_back(last_kps[idx].angle);
        has_obs.push_back(lm->has_observation() ? 1 : 0);
        table.push_back(lm);
    }

    b200_track_params_t prm{};
    fill_track_params(curr_frm, prm);
    const auto* cam = curr_frm.camera_;
    prm.margin = margin;       // margin_last_frame_projection
    prm.lowe_ratio = 0.9f;     // match::projection projection_matcher(0.9, true) (:21); mode 1 has no ratio test
    prm.hamming_thr = 100;     // HAMMING_DIST_THR_HIGH

    const Mat44_t pose_cw = velocity * last_frm.get_pose_cw();  // :24
    const Mat44_t last_pose_cw = last_frm.get_pose_cw();
    double pose[16], last_pose[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            pose[4 * r + c] = pose_cw(r, c);
            last_pose[4 * r + c] = last_pose_cw(r, c);
        }
    const unsigned int num_keypts = curr_frm.frm_obs_.undist_keypts_.size();
    std::vector<int32_t> kp_landmark_out(num_keypts + 1, -1);
    b200_motion_track_frame_t f{};
    f.frame = 0;
    f.pose_cw = pose;
    f.last_pose_cw = last_pose;
    const bool stereo = !curr_frm.frm_obs_.stereo_x_right_.empty();
    f.n_keypoints_in = stereo ? static_cast<int32_t>(num_keypts) : 0;
    f.kp_x_right = stereo ? curr_frm.frm_obs_.stereo_x_right_.data() : nullptr;
    f.n_landmarks = static_cast<int32_t>(table.size());
    f.lm_pos_w = pos.data(); f.lm_desc = desc.data(); f.lm_octave = octave.data(); f.lm_angle = angle.data(); f.lm_has_observation = has_obs.data();
    f.kp_cap = static_cast<int32_t>(num_keypts);
    f.kp_landmark_out = kp_landmark_out.data();
    if (b200_motion_based_track(orb, matcher, opt, &prm, cam->true_baseline_, num_matches_thr, 1, &f) != B200_OK)
        throw std::runtime_error(b200_last_error());
    if (static_cast<unsigned int>(f.n_keypoints) != num_keypts) throw std::runtime_error("motion_based_track_b200: the extractor's last frame is not curr_frm");

    // ---- write-back: the frame starts without landmarks (:27) and carries what survived the search and discard_outliers
    curr_frm.erase_landmarks();
    for (unsigned int idx = 0; idx < num_keypts; ++idx)
        if (kp_landmark_out[idx] >= 0) curr_frm.add_landmark(table[kp_landmark_out[idx]], idx);
    Mat44_t out;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) out(r, c) = f.pose_cw_out[4 * r + c];
    curr_frm.set_pose_cw(out);
    return f.tracked != 0;
}

// module::frame_tracker::robust_match_based_track (module/frame_tracker.cc:97-131) as one device call: brute-force match against the
// reference keyframe, the five-point RANSAC with its minimal sets drawn on the device, set_landmarks, the pose optimisation from the last
// pose and discard_outliers (b200_robust_match_based_track).  Only the keyframe's side goes up; the frame's keypoints and descriptors are
// read where the GPU extractor left them.
// Call site (tracking_module::track_current_frame, tracking_module.cc:333-355, USE_B200), in place of the robust fallback:
//     succeeded = frame_tracker_.robust_match_based_track(curr_frm_, last_frm_, curr_frm_.ref_keyfrm_);
//         -> succeeded = robust_match_based_track_b200(curr_frm_, last_frm_, curr_frm_.ref_keyfrm_, extractor_left_, use_fixed_seed_,
//                                                      num_matches_thr);
// Precondition as motion_based_track_b200.  Returns what frame_tracker::robust_match_based_track returns; curr_frm is left exactly as it
// was when the frame is not applied (fewer inliers than num_matches_thr, :105-108).
bool robust_match_based_track_b200(data::frame& curr_frm, const data::frame& last_frm, const std::shared_ptr<data::keyframe>& ref_keyfrm,
                                   const feature::orb_extractor* extractor, bool use_fixed_seed, unsigned int num_matches_thr) {
    const b200_orb_t orb = feature::b200_handle_of(extractor);
    if (!orb) throw std::runtime_error("robust_match_based_track_b200: the extractor has not extracted a frame yet");
    static thread_local b200_matcher_t matcher = nullptr;
    static thread_local b200_lba_t opt = nullptr;
    if (!matcher && b200_matcher_create(0, &matcher) != B200_OK) throw std::runtime_error(b200_last_error());
    if (!opt && b200_lba_create(0, &opt) != B200_OK) throw std::runtime_error(b200_last_error());

    // ---- the keyframe side, in keyframe keypoint order; the same landmark vector serves the write-back (robust.cc:201, 243)
    const auto keyfrm_lms = ref_keyfrm->get_landmarks();
    const auto& kf_kps = ref_keyfrm->frm_obs_.undist_keypts_;
    const unsigned int n_kf = kf_kps.size();
    std::vector<float> kf_angle(n_kf);
    std::vector<uint8_t> kf_valid(n_kf, 0);
    std::vector<double> kf_pos(3 * (size_t)n_kf, 0.0);
    for (unsigned int i = 0; i < n_kf; ++i) {
        kf_angle[i] = kf_kps[i].angle;
        const auto& lm = keyfrm_lms.at(i);
        if (!lm || lm->will_be_erased()) continue;  // robust.cc:255-262
        kf_valid[i] = 1;
        const Vec3_t p = lm->get_pos_in_world();
        kf_pos[3 * i] = p(0); kf_pos[3 * i + 1] = p(1); kf_pos[3 * i + 2] = p(2);
    }
    std::vector<double> kf_bearings(3 * (size_t)n_kf);
    for (unsigned int i = 0; i < n_kf; ++i)
        for (int k = 0; k < 3; ++k) kf_bearings[3 * i + k] = ref_keyfrm->frm_obs_.bearings_.at(i)(k);

    b200_track_params_t prm{};
    fill_track_params(curr_frm, prm);
    prm.lowe_ratio = 0.8f;  // match::robust robust_matcher(0.8, true) (:98)

    // util::create_random_engine(use_fixed_seed): a default-constructed engine (NULL), or std::seed_seq over ten std::random_device words
    b200_mt19937_t engine;
    if (!use_fixed_seed) {
        std::random_device rd;
        uint32_t words[10];
        for (auto& w : words) w = rd();
        b200_mt19937_seed(&engine, words, 10);
    }

    const Mat44_t last_pose_cw = last_frm.get_pose_cw();  // :115
    double last_pose[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) last_pose[4 * r + c] = last_pose_cw(r, c);
    const unsigned int num_keypts = curr_frm.frm_obs_.undist_keypts_.size();
    std::vector<int32_t> kp_landmark_out(num_keypts + 1, -1);
    b200_robust_track_frame_t f{};
    f.frame = 0;
    f.last_pose_cw = last_pose;
    const bool stereo = !curr_frm.frm_obs_.stereo_x_right_.empty();
    f.n_keypoints_in = stereo ? static_cast<int32_t>(num_keypts) : 0;
    f.kp_x_right = stereo ? curr_frm.frm_obs_.stereo_x_right_.data() : nullptr;
    f.engine = use_fixed_seed ? nullptr : &engine;
    f.n_kf_keypoints = static_cast<int32_t>(n_kf);
    f.kf_desc = ref_keyfrm->frm_obs_.descriptors_.ptr<uint8_t>();
    f.kf_angle = kf_angle.data();
    f.kf_bearings = kf_bearings.data();
    f.kf_valid = kf_valid.data();
    f.kf_pos_w = kf_pos.data();
    f.kp_cap = static_cast<int32_t>(num_keypts);
    f.kp_landmark_out = kp_landmark_out.data();
    if (b200_robust_match_based_track(orb, matcher, opt, &prm, num_matches_thr, 1, &f) != B200_OK) throw std::runtime_error(b200_last_error());
    if (static_cast<unsigned int>(f.n_keypoints) != num_keypts)
        throw std::runtime_error("robust_match_based_track_b200: the extractor's last frame is not curr_frm");
    if (!f.applied) return false;  // :105-108: the frame is not touched

    // ---- write-back: set_landmarks (:111) with the landmarks that survived discard_outliers, then the optimised pose
    std::vector<std::shared_ptr<data::landmark>> lms(num_keypts, nullptr);
    for (unsigned int idx = 0; idx < num_keypts; ++idx)
        if (kp_landmark_out[idx] >= 0) lms[idx] = keyfrm_lms.at(kp_landmark_out[idx]);
    curr_frm.set_landmarks(lms);
    Mat44_t out;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) out(r, c) = f.pose_cw_out[4 * r + c];
    curr_frm.set_pose_cw(out);
    return f.tracked != 0;
}

// module::frame_tracker::bow_match_based_track (module/frame_tracker.cc:61-95) as one device call: bow_tree(0.7, true)::
// match_frame_and_keyframe against the reference keyframe, the gate, set_landmarks, the pose optimisation from the last pose and
// discard_outliers (b200_bow_match_based_track).  The BoW vectors stay on the host: only one node id per keypoint on each side, and the
// keyframe's descriptors, angles and landmark positions go up; the frame's keypoints and descriptors are read where the GPU extractor
// left them.
// Call site (tracking_module::track_current_frame, tracking_module.cc:333-355, USE_B200), in place of the first fallback, after
// curr_frm_.compute_bow(bow_vocab_) (:343-345):
//     succeeded = frame_tracker_.bow_match_based_track(curr_frm_, last_frm_, curr_frm_.ref_keyfrm_);
//         -> succeeded = bow_match_based_track_b200(curr_frm_, last_frm_, curr_frm_.ref_keyfrm_, extractor_left_, num_matches_thr);
// Precondition as motion_based_track_b200, and both bow_feat_vec_ computed.  Returns what frame_tracker::bow_match_based_track returns;
// curr_frm is left exactly as it was when the frame is not applied (fewer matches than num_matches_thr, :69-72).
bool bow_match_based_track_b200(data::frame& curr_frm, const data::frame& last_frm, const std::shared_ptr<data::keyframe>& ref_keyfrm,
                                const feature::orb_extractor* extractor, unsigned int num_matches_thr) {
    const b200_orb_t orb = feature::b200_handle_of(extractor);
    if (!orb) throw std::runtime_error("bow_match_based_track_b200: the extractor has not extracted a frame yet");
    static thread_local b200_matcher_t matcher = nullptr;
    static thread_local b200_lba_t opt = nullptr;
    if (!matcher && b200_matcher_create(0, &matcher) != B200_OK) throw std::runtime_error(b200_last_error());
    if (!opt && b200_lba_create(0, &opt) != B200_OK) throw std::runtime_error(b200_last_error());

    // ---- the keyframe side, in keyframe keypoint order; the same landmark vector serves the write-back (bow_tree.cc:174, 247)
    const auto keyfrm_lms = ref_keyfrm->get_landmarks();
    const auto& kf_kps = ref_keyfrm->frm_obs_.undist_keypts_;
    const unsigned int n_kf = kf_kps.size();
    std::vector<float> kf_angle(n_kf);
    std::vector<uint8_t> kf_valid(n_kf, 0);
    std::vector<double> kf_pos(3 * (size_t)n_kf, 0.0);
    for (unsigned int i = 0; i < n_kf; ++i) {
        kf_angle[i] = kf_kps[i].angle;
        const auto& lm = keyfrm_lms.at(i);
        if (!lm || lm->will_be_erased()) continue;  // bow_tree.cc:192-199
        kf_valid[i] = 1;
        const Vec3_t p = lm->get_pos_in_world();
        kf_pos[3 * i] = p(0); kf_pos[3 * i + 1] = p(1); kf_pos[3 * i + 2] = p(2);
    }
    const unsigned int num_keypts = curr_frm.frm_obs_.undist_keypts_.size();
    const auto kf_node = b200_gather::node_of(ref_keyfrm->bow_feat_vec_, n_kf);
    const auto kp_node = b200_gather::node_of(curr_frm.bow_feat_vec_, num_keypts);

    b200_track_params_t prm{};
    fill_track_params(curr_frm, prm);
    prm.lowe_ratio = 0.7f;  // match::bow_tree bow_matcher(0.7, true) (:62)

    const Mat44_t last_pose_cw = last_frm.get_pose_cw();  // :78
    double last_pose[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) last_pose[4 * r + c] = last_pose_cw(r, c);
    std::vector<int32_t> kp_landmark_out(num_keypts + 1, -1);
    b200_bow_track_frame_t f{};
    f.frame = 0;
    f.last_pose_cw = last_pose;
    f.n_keypoints_in = static_cast<int32_t>(num_keypts);
    f.kp_node = kp_node.data();
    const bool stereo = !curr_frm.frm_obs_.stereo_x_right_.empty();
    f.kp_x_right = stereo ? curr_frm.frm_obs_.stereo_x_right_.data() : nullptr;
    f.n_kf_keypoints = static_cast<int32_t>(n_kf);
    f.kf_desc = ref_keyfrm->frm_obs_.descriptors_.ptr<uint8_t>();
    f.kf_angle = kf_angle.data();
    f.kf_node = kf_node.data();
    f.kf_valid = kf_valid.data();
    f.kf_pos_w = kf_pos.data();
    f.kp_cap = static_cast<int32_t>(num_keypts);
    f.kp_landmark_out = kp_landmark_out.data();
    if (b200_bow_match_based_track(orb, matcher, opt, &prm, num_matches_thr, 1, &f) != B200_OK) throw std::runtime_error(b200_last_error());
    if (!f.applied) return false;  // :69-72: the frame is not touched

    // ---- write-back: set_landmarks (:75) with the landmarks that survived discard_outliers, then the optimised pose
    std::vector<std::shared_ptr<data::landmark>> lms(num_keypts, nullptr);
    for (unsigned int idx = 0; idx < num_keypts; ++idx)
        if (kp_landmark_out[idx] >= 0) lms[idx] = keyfrm_lms.at(kp_landmark_out[idx]);
    curr_frm.set_landmarks(lms);
    Mat44_t out;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) out(r, c) = f.pose_cw_out[4 * r + c];
    curr_frm.set_pose_cw(out);
    return f.tracked != 0;
}

}  // namespace stella_vslam
