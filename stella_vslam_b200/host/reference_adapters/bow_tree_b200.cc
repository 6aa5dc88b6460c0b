// Replacement bodies for the three BoW matchers
//   match::bow_tree::match_for_triangulation   (src/stella_vslam/match/bow_tree.cc:11-167)
//   match::bow_tree::match_frame_and_keyframe  (bow_tree.cc:169-256)
//   match::bow_tree::match_keyframes           (bow_tree.cc:258-366)
// and for match::robust::match_for_triangulation (src/stella_vslam/match/robust.cc:14-146), which is the same matcher without the BoW
// gate.  Guard the originals with #ifndef USE_B200.  The reference's merge-join over the two bow_feat_vec_ maps pairs the keypoints that
// fall into the same vocabulary node; a keypoint belongs to exactly one node, rows of different nodes never compete for a candidate
// and the index lists of a node are ascending (compute_bow walks the descriptors in order), so "row i sees candidate j iff
// node[i] == node[j], rows in index order" reproduces it -- that is the gate b200_match_pairs applies.
#include <stdexcept>

#include "stella_vslam/camera/base.h"
#include "stella_vslam/data/bow_vocabulary.h"
#include "stella_vslam/data/frame.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/match/bow_tree.h"
#include "stella_vslam/match/robust.h"

#include "b200vslam.h"
#include "pairs_gather_b200.h"

namespace stella_vslam {
namespace match {
namespace {

b200_matcher_t pairs_matcher() {
    static thread_local b200_matcher_t h = nullptr;
    if (!h && b200_matcher_create(0, &h) != B200_OK) throw std::runtime_error(b200_last_error());
    return h;
}

using b200_gather::node_of;
using b200_gather::side;

// shared body of the two match_for_triangulation (robust.cc:14-146, bow_tree.cc:11-167)
unsigned int triangulation(const std::shared_ptr<data::keyframe>& keyfrm_1, const std::shared_ptr<data::keyframe>& keyfrm_2, const Mat33_t& E_12,
                           std::vector<std::pair<unsigned int, unsigned int>>& matched_idx_pairs, const float residual_rad_thr, bool bow, float lowe_ratio,
                           bool check_orientation) {
    const Vec3_t cam_center_1 = keyfrm_1->get_trans_wc();
    Vec3_t epiplane_in_keyfrm_2;
    const bool valid_epiplane = keyfrm_2->camera_->reproject_to_bearing(keyfrm_2->get_rot_cw(), keyfrm_2->get_trans_cw(), cam_center_1, epiplane_in_keyfrm_2);
    const auto lms_1 = keyfrm_1->get_landmarks();
    const auto lms_2 = keyfrm_2->get_landmarks();
    side s1, s2;
    s1.fill(keyfrm_1->frm_obs_, keyfrm_1->orb_params_);
    s2.fill(keyfrm_2->frm_obs_, keyfrm_2->orb_params_);
    for (size_t i = 0; i < s1.valid.size(); ++i) s1.valid[i] = !lms_1.at(i);  // only keypoints WITHOUT a landmark (robust.cc:44-48)
    for (size_t i = 0; i < s2.valid.size(); ++i) s2.valid[i] = !lms_2.at(i);  // (:66-69)
    std::vector<int32_t> node1, node2, out(s1.valid.size(), -1);
    if (bow) {
        node1 = node_of(keyfrm_1->bow_feat_vec_, s1.valid.size());
        node2 = node_of(keyfrm_2->bow_feat_vec_, s2.valid.size());
    }
    b200_pairs_problem_t P{};
    P.n1 = static_cast<int32_t>(s1.valid.size());
    P.desc1 = keyfrm_1->frm_obs_.descriptors_.data; P.angle1 = s1.angle.data(); P.valid1 = s1.valid.data(); P.node1 = bow ? node1.data() : nullptr;
    P.bearing1 = s1.bearing.data(); P.scale1 = s1.scale.data(); P.stereo1 = s1.stereo.data();
    P.n2 = static_cast<int32_t>(s2.valid.size());
    P.desc2 = keyfrm_2->frm_obs_.descriptors_.data; P.angle2 = s2.angle.data(); P.valid2 = s2.valid.data(); P.node2 = bow ? node2.data() : nullptr;
    P.bearing2 = s2.bearing.data(); P.stereo2 = s2.stereo.data();
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) P.E_12[3 * r + c] = E_12(r, c);
    for (int k = 0; k < 3; ++k) P.epiplane_in_keyfrm_2[k] = epiplane_in_keyfrm_2(k);
    P.valid_epiplane = valid_epiplane ? 1 : 0;
    P.residual_rad_thr = residual_rad_thr;
    P.match_out = out.data();
    if (b200_match_pairs(pairs_matcher(), 1, &P, B200_PAIRS_TRIANGULATION, lowe_ratio, check_orientation ? 1 : 0, 0) != B200_OK)
        throw std::runtime_error(b200_last_error());
    matched_idx_pairs.clear();
    matched_idx_pairs.reserve(P.n_matches);
    for (unsigned int idx_1 = 0; idx_1 < out.size(); ++idx_1)  // :136-143
        if (0 <= out[idx_1]) matched_idx_pairs.emplace_back(std::make_pair(idx_1, static_cast<unsigned int>(out[idx_1])));
    return static_cast<unsigned int>(P.n_matches);
}

}  // namespace

unsigned int bow_tree::match_for_triangulation(const std::shared_ptr<data::keyframe>& keyfrm_1, const std::shared_ptr<data::keyframe>& keyfrm_2,
                                               const Mat33_t& E_12, std::vector<std::pair<unsigned int, unsigned int>>& matched_idx_pairs,
                                               const float residual_rad_thr) const {
    return triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs, residual_rad_thr, true, lowe_ratio_, check_orientation_);
}

unsigned int robust::match_for_triangulation(const std::shared_ptr<data::keyframe>& keyfrm_1, const std::shared_ptr<data::keyframe>& keyfrm_2,
                                             const Mat33_t& E_12, std::vector<std::pair<unsigned int, unsigned int>>& matched_idx_pairs,
                                             const float residual_rad_thr) const {
    return triangulation(keyfrm_1, keyfrm_2, E_12, matched_idx_pairs, residual_rad_thr, false, lowe_ratio_, check_orientation_);
}

// bow_tree.cc:169-256: rows = keyframe keypoints with a live landmark, candidates = frame keypoints that have not received one yet
unsigned int bow_tree::match_frame_and_keyframe(const std::shared_ptr<data::keyframe>& keyfrm, data::frame& frm,
                                                std::vector<std::shared_ptr<data::landmark>>& matched_lms_in_frm) const {
    const size_t n_frm = frm.frm_obs_.undist_keypts_.size();
    matched_lms_in_frm = std::vector<std::shared_ptr<data::landmark>>(n_frm, nullptr);
    const auto keyfrm_lms = keyfrm->get_landmarks();
    side s1, s2;
    s1.fill(keyfrm->frm_obs_, keyfrm->orb_params_);
    s2.fill(frm.frm_obs_, frm.orb_params_);
    for (size_t i = 0; i < s1.valid.size(); ++i) s1.valid[i] = keyfrm_lms.at(i) && !keyfrm_lms.at(i)->will_be_erased();  // :192-199
    const auto node1 = node_of(keyfrm->bow_feat_vec_, s1.valid.size());
    const auto node2 = node_of(frm.bow_feat_vec_, n_frm);
    std::vector<int32_t> out(s1.valid.size(), -1);
    b200_pairs_problem_t P{};
    P.n1 = static_cast<int32_t>(s1.valid.size());
    P.desc1 = keyfrm->frm_obs_.descriptors_.data; P.angle1 = s1.angle.data(); P.valid1 = s1.valid.data(); P.node1 = node1.data();
    P.n2 = static_cast<int32_t>(n_frm);
    P.desc2 = frm.frm_obs_.descriptors_.data; P.angle2 = s2.angle.data(); P.valid2 = nullptr; P.node2 = node2.data();
    P.match_out = out.data();
    if (b200_match_pairs(pairs_matcher(), 1, &P, B200_PAIRS_BOW, lowe_ratio_, check_orientation_ ? 1 : 0, 0) != B200_OK)
        throw std::runtime_error(b200_last_error());
    for (size_t i = 0; i < out.size(); ++i)
        if (0 <= out[i]) matched_lms_in_frm.at(out[i]) = keyfrm_lms.at(i);  // :239
    return static_cast<unsigned int>(P.n_matches);
}

// bow_tree.cc:258-366: both sides need a live landmark
unsigned int bow_tree::match_keyframes(const std::shared_ptr<data::keyframe>& keyfrm_1, const std::shared_ptr<data::keyframe>& keyfrm_2,
                                       std::vector<std::shared_ptr<data::landmark>>& matched_lms_in_keyfrm_1) const {
    const auto lms_1 = keyfrm_1->get_landmarks();
    const auto lms_2 = keyfrm_2->get_landmarks();
    matched_lms_in_keyfrm_1 = std::vector<std::shared_ptr<data::landmark>>(lms_1.size(), nullptr);
    side s1, s2;
    s1.fill(keyfrm_1->frm_obs_, keyfrm_1->orb_params_);
    s2.fill(keyfrm_2->frm_obs_, keyfrm_2->orb_params_);
    for (size_t i = 0; i < s1.valid.size(); ++i) s1.valid[i] = lms_1.at(i) && !lms_1.at(i)->will_be_erased();  // :284-291
    for (size_t i = 0; i < s2.valid.size(); ++i) s2.valid[i] = lms_2.at(i) && !lms_2.at(i)->will_be_erased();  // :303-309
    const auto node1 = node_of(keyfrm_1->bow_feat_vec_, s1.valid.size());
    const auto node2 = node_of(keyfrm_2->bow_feat_vec_, s2.valid.size());
    std::vector<int32_t> out(s1.valid.size(), -1);
    b200_pairs_problem_t P{};
    P.n1 = static_cast<int32_t>(s1.valid.size());
    P.desc1 = keyfrm_1->frm_obs_.descriptors_.data; P.angle1 = s1.angle.data(); P.valid1 = s1.valid.data(); P.node1 = node1.data();
    P.n2 = static_cast<int32_t>(s2.valid.size());
    P.desc2 = keyfrm_2->frm_obs_.descriptors_.data; P.angle2 = s2.angle.data(); P.valid2 = s2.valid.data(); P.node2 = node2.data();
    P.match_out = out.data();
    if (b200_match_pairs(pairs_matcher(), 1, &P, B200_PAIRS_BOW, lowe_ratio_, check_orientation_ ? 1 : 0, 0) != B200_OK)
        throw std::runtime_error(b200_last_error());
    for (size_t i = 0; i < out.size(); ++i)
        if (0 <= out[i]) matched_lms_in_keyfrm_1.at(i) = lms_2.at(out[i]);  // :349
    return static_cast<unsigned int>(P.n_matches);
}

}  // namespace match
}  // namespace stella_vslam
